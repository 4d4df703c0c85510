"""Sequential CPU model of the batched GPU build (test infrastructure).

The GPU builder (embeddinghub_b200/csrc/build_impl.cuh) links points in waves.  This module restates what one wave
computes, over a precomputed exact distance matrix, so that on data whose distances are exact and free of ties the
GPU graph must equal the model's row for row, in order.  The rules (also in DESIGN.md, K5 construction):

Inserts.  A wave holds points [n_linked, n_linked + b) with b = min(build_batch or 16384, max(1, n_linked //
(build_frac or 64)), n - n_linked); the first point is linked alone.  Every point of a wave reads the graph as it was
when the wave started.
  phase A: greedy descent from the entry over the layers above the point's level, then per layer min(level,
    max_level) .. 0 hnswlib's construction beam search (efc = max(ef_construction, M); results by (distance, id); an
    empty layer is skipped), getNeighborsByHeuristic2 with M; the selection, in order, is the point's row; the next
    layer starts from this layer's closest result.  One (target row, source, distance) record per selected neighbour.
  phase C: per touched row, the records in source-id order: a source the row holds is skipped; one is appended while
    the row has room; a full row is re-selected over (row + source): the 128 closest by (distance, id), then the
    heuristic with W (M0 at layer 0, M above).  After the 4th re-selection every record not yet applied is folded
    into that same re-selection, and the row is done.  Rows keep selection order, then append order.
  After the wave the first point of the highest level above max_level (ascending id) becomes the entry.

Updates.  Moved points in first-arrival order (each with the last vector written); one point per wave while at most
`seq_updates` (4096 by default) are pending, else waves of build_batch or 1024.  One wave:
  U1: per moved point p and layer <= its level, sCand = {p} + one-hop(p) + two-hop(p) from the pre-wave graph; the
    row of each one-hop neighbour nb is re-selected over sCand - {nb}: keep min(efc, |sCand| - 1), then Mmax.  When
    several moved points re-select one row the latest in arrival order wins; all re-selections land together.
  U2: each moved point is re-linked as in phase A over the graph after U1; the point itself is walked and admitted
    like any other node and dropped from each layer's result list before the selection (hnswlib
    repairConnectionsForUpdate).  Its own rows are replaced together, then phase C runs as above.

Tombstones are traversed but never results (hnswlib's construction searchBaseLayer).
"""
import heapq

import numpy as np

from compact_model import _reselect

INV = 0xFFFFFFFF
MERGE_KEEP = 128          # the re-selection keeps this many candidates before the heuristic (cfg.lcap)
MAX_SEQ_PRUNES = 3        # re-selections applied one record at a time before the rest is folded
SEQ_UPDATES = 4096        # default: up to this many pending moves go one point per wave


class WaveModel:
    """The graph of one index under the wave rules.  D: exact distances ([n][n], D[a][b] = D[b][a]); levels: level
    of every point (the index's level generator decides them; tests take them from the index)."""

    def __init__(self, D, levels, M, ef_construction=200):
        self.set_distances(D)
        self.levels = [int(v) for v in levels]
        self.n = len(self.levels)
        self.M, self.M0 = int(M), 2 * int(M)
        self.efc = max(int(ef_construction), self.M)
        self.deleted = set()
        self.rows = [[[] for _ in range(lv + 1)] for lv in self.levels]
        self.n_linked = 0
        self.entry, self.max_level = 0, -1
        # trace: the largest number of records one row received in a wave, phase-C re-selections, folds, folds
        # of rows that received more than MERGE_KEEP records (the hub case), wave sizes
        self.trace = {"max_incoming": 0, "reselects": 0, "folds": 0, "hub_folds": 0, "waves": []}

    def set_distances(self, D):
        """New exact distances (after moves: every moved point's last vector)."""
        D = np.asarray(D, np.float64)
        self.D = D.tolist()                                      # rows as lists: the searches index them per id
        self.dist = lambda i, ids: D[i, ids]

    def mark_deleted(self, ids):
        self.deleted.update(int(i) for i in ids)

    # ---- graph access -------------------------------------------------------------------------------------
    def row(self, p, layer):
        return self.rows[p][layer]

    def export(self):
        """The graph in the index's export layout: links0 [n][M0], up_off [n] (INV at level 0), links_up, entry,
        maxlevel."""
        n, M, M0 = self.n, self.M, self.M0
        links0 = np.full((n, M0), INV, np.uint32)
        up_off = np.full(n, INV, np.uint32)
        up = []
        for p in range(n):
            r = self.rows[p][0]
            links0[p, :len(r)] = r
            if self.levels[p]:
                up_off[p] = len(up)
                for layer in range(1, self.levels[p] + 1):
                    row = np.full(M, INV, np.uint32)
                    r = self.rows[p][layer]
                    row[:len(r)] = r
                    up.append(row)
        return {"levels": np.asarray(self.levels, np.uint8), "links0": links0, "up_off": up_off,
                "links_up": np.asarray(up, np.uint32).reshape(-1, M), "entry": self.entry,
                "maxlevel": self.max_level}

    def load(self, g, n_linked):
        """Adopt an exported graph of the first n_linked points (the rest stay unlinked)."""
        self.n_linked = int(n_linked)
        self.entry, self.max_level = int(g["entry"]), int(g["maxlevel"])
        for p in range(self.n_linked):
            self.rows[p][0] = [int(v) for v in g["links0"][p] if v != INV]
            for layer in range(1, self.levels[p] + 1):
                r = g["links_up"][int(g["up_off"][p]) + layer - 1]
                self.rows[p][layer] = [int(v) for v in r if v != INV]

    # ---- searches -----------------------------------------------------------------------------------------
    def _greedy(self, dl, cur, top, bottom_excl):
        cd = dl[cur]
        for layer in range(top, bottom_excl, -1):
            changed = True
            while changed:
                changed = False
                for nb in self.rows[cur][layer]:
                    if dl[nb] < cd:
                        cd, cur, changed = dl[nb], nb, True
        return cur

    def _search(self, dl, ep, layer):
        """hnswlib searchBaseLayer: ascending (distance, id) list of <= efc results."""
        efc, deleted, rows = self.efc, self.deleted, self.rows
        visited = {ep}
        top = []                              # max-heap of (-d, -id)
        cand = []                             # min-heap of (d, id)
        if ep in deleted:
            lower = float("inf")
        else:
            lower = dl[ep]
            top.append((-lower, -ep))
        cand.append((dl[ep] if top else float("-inf"), ep))
        while cand:
            d, c = heapq.heappop(cand)
            if d > lower and len(top) == efc:
                break
            for nb in rows[c][layer]:
                if nb in visited:
                    continue
                visited.add(nb)
                dd = dl[nb]
                if len(top) < efc or lower > dd:
                    heapq.heappush(cand, (dd, nb))
                    if nb not in deleted:
                        heapq.heappush(top, (-dd, -nb))
                        if len(top) > efc:
                            heapq.heappop(top)
                    if top:
                        lower = -top[0][0]
        return [-i for _, i in sorted(top, key=lambda t: (-t[0], -t[1]))]

    def _link(self, p, exclude_self):
        """Phase A for one point: {layer: selected row} and the reverse-edge records [(layer, target, source)]."""
        dl = self.D[p]
        lp = self.levels[p]
        cur = self.entry
        if lp < self.max_level:
            cur = self._greedy(dl, cur, self.max_level, lp)
        out, recs = {}, []
        for layer in range(min(lp, self.max_level), -1, -1):
            res = self._search(dl, cur, layer)
            if exclude_self:                  # repairConnectionsForUpdate: searched like any node, then dropped
                res = [v for v in res if v != p]
            if not res:
                continue
            sel = _reselect(p, res, self.dist, len(res), self.M)
            out[layer] = sel
            recs.extend((layer, t, p) for t in sel)
            cur = res[0]
        return out, recs

    # ---- phase C --------------------------------------------------------------------------------------------
    def _merge(self, recs):
        by_row = {}
        for layer, t, s in recs:
            by_row.setdefault((layer, t), []).append(s)
        for (layer, t), srcs in by_row.items():
            srcs.sort()
            self.trace["max_incoming"] = max(self.trace["max_incoming"], len(srcs))
            W = self.M0 if layer == 0 else self.M
            row = list(self.rows[t][layer])
            prunes = 0
            for i, s in enumerate(srcs):
                if s in row:
                    continue
                if len(row) < W:
                    row.append(s)
                    continue
                cand = set(row)
                cand.add(s)
                prunes += 1
                self.trace["reselects"] += 1
                fold = prunes > MAX_SEQ_PRUNES
                if fold:
                    cand.update(srcs[i + 1:])
                    self.trace["folds"] += 1
                    if len(srcs) > MERGE_KEEP:
                        self.trace["hub_folds"] += 1
                row = _reselect(t, cand, self.dist, MERGE_KEEP, W)
                if fold:
                    break
            self.rows[t][layer] = row

    # ---- inserts --------------------------------------------------------------------------------------------
    def insert_wave(self, b):
        lo = self.n_linked
        if lo == 0:
            self.entry, self.max_level, self.n_linked = 0, self.levels[0], 1
            self.trace["waves"].append(1)
            return
        own, recs = {}, []
        for p in range(lo, lo + b):
            own[p], r = self._link(p, False)
            recs.extend(r)
        for p, sel in own.items():
            for layer, r in sel.items():
                self.rows[p][layer] = r
        self._merge(recs)
        for p in range(lo, lo + b):
            if self.levels[p] > self.max_level:
                self.max_level, self.entry = self.levels[p], p
        self.n_linked = lo + b
        self.trace["waves"].append(b)

    def build(self, n=None, build_batch=0, build_frac=0):
        n = self.n if n is None else int(n)
        maxb = build_batch or 16384
        frac = build_frac or 64
        while self.n_linked < n:
            if self.n_linked == 0:
                self.insert_wave(1)
                continue
            b = min(maxb, max(1, self.n_linked // frac), n - self.n_linked)
            self.insert_wave(b)
        return self

    # ---- updates --------------------------------------------------------------------------------------------
    def update_wave(self, ids):
        staged = {}
        for p in ids:
            for layer in range(min(self.levels[p], self.max_level) + 1):
                one = self.rows[p][layer]
                if not one:
                    continue
                scand = {p}
                scand.update(one)
                for e1 in one:
                    scand.update(self.rows[e1][layer])
                mmax = self.M0 if layer == 0 else self.M
                keep = min(self.efc, len(scand) - 1)
                for nb in one:
                    staged[(nb, layer)] = _reselect(nb, scand - {nb}, self.dist, keep, mmax)   # later arrivals win
        for (nb, layer), r in staged.items():
            self.rows[nb][layer] = r
        own, recs = {}, []
        for p in ids:
            own[p], r = self._link(p, True)
            recs.extend(r)
        for p, sel in own.items():
            for layer, r in sel.items():
                self.rows[p][layer] = r
        self._merge(recs)

    def update(self, moved, build_batch=0, seq_updates=SEQ_UPDATES):
        """moved: ids in arrival order (repeats allowed); the distance matrix must already hold the final
        vectors."""
        ups, seen = [], set()
        for p in moved:
            p = int(p)
            if p not in seen:
                seen.add(p)
                ups.append(p)
        if self.n_linked <= 1:
            return self
        ub = 1 if len(ups) <= seq_updates else (build_batch or 1024)
        for off in range(0, len(ups), ub):
            self.update_wave(ups[off:off + ub])
        return self


# ---- exact data -----------------------------------------------------------------------------------------------
def tiefree_ip(n, d, seed=11, nnz=None):
    """Build-tie-free inner-product rows x_i = (B u_i, i + 1), B = 2^bitlen(n) > n + 1, so x_a.x_b = B^2 (u_a.u_b) +
    (a+1)(b+1) is exact and distinct over b.  u_i in {-1, 0, 1}^(d-1), dense when nnz is None, else with nnz
    non-zeros spread over all d - 1 coordinates; every partial sum stays below B^2 nnz + (n+1)^2 < 2^24, so any
    summation order gives the same fp32 value."""
    B = 1 << n.bit_length()
    rng = np.random.default_rng(seed)
    x = np.zeros((n, d), np.int64)
    if nnz is None:
        x[:, :d - 1] = B * rng.integers(-1, 2, (n, d - 1))
        nnz = d - 1
    else:
        for i in range(n):
            cols = rng.choice(d - 1, nnz, replace=False)
            x[i, cols] = B * rng.choice([-1, 1], nnz)
    x[:, d - 1] = np.arange(1, n + 1)
    assert B * B * nnz + (n + 1) ** 2 < 1 << 24
    return x, B


def hub_ip(n, d):
    """x_i = (i + 1) e_{d-1}: every point orders all others the same way (highest id first); exact for n <= 4095."""
    assert (n + 1) ** 2 < 1 << 24
    x = np.zeros((n, d), np.int64)
    x[:, d - 1] = np.arange(1, n + 1)
    return x


def ip_matrix(x):
    """Exact 1 - x_a.x_b for integer rows."""
    x = np.asarray(x, np.int64)
    D = 1 - x @ x.T
    assert np.abs(D).max() < 1 << 24
    return D.astype(np.float64)
