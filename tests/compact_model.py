"""Sequential CPU model of ehb_index_compact (test infrastructure).

Steps 1-4 and 6 of the compaction are restated here in numpy; step 5 (re-linking the orphans) is the oracle's own
updatePoint, reached the way hnswlib reaches it: re-adding an existing label with its vector.  Every step reads
the pre-compaction graph, exactly as the GPU passes do, so the model and the GPU agree row for row wherever the
distances are exact and free of ties.
"""
import numpy as np

from oracle import oracle as orc  # test infrastructure

INV = 0xFFFFFFFF


def _row(g, p, layer):
    r = g["links0"][p] if layer == 0 else g["links_up"][int(g["up_off"][p]) + layer - 1]
    return [int(v) for v in r if v != INV]


def _reselect(p, cand, dist, keep, mmax):
    """The keep-then-select step of hnswlib updatePoint: the `keep` candidates closest to p, ordered by
    (distance, id), then getNeighborsByHeuristic2 with mmax."""
    ids = np.asarray(sorted(cand), np.int64)
    d = dist(p, ids)
    order = np.lexsort((ids, d))[:keep]
    ids, d = ids[order], d[order]
    if len(ids) < mmax:
        return ids.tolist()
    kept = []
    for i, c in enumerate(ids.tolist()):
        if len(kept) >= mmax:
            break
        if not kept or not np.any(dist(c, np.asarray(kept, np.int64)) < d[i]):
            kept.append(c)
    return kept


def compact_graph(g, dead, dist, M, efc):
    """Steps 1-4 and 6 on an exported graph.  dead: bool per internal id; dist(i, ids) -> distances from row i
    to rows ids.  Returns (compacted graph dict, orphan ids in the new numbering)."""
    n = len(g["levels"])
    dead = np.asarray(dead, bool)
    live = np.flatnonzero(~dead)
    M0 = 2 * M
    levels = np.asarray(g["levels"]).astype(np.int64)
    # 1 + 2. rows of live nodes that name deleted ids, re-selected over the pre-compaction graph
    repaired = {}
    for p in live.tolist():
        for layer in range(levels[p] + 1):
            r = _row(g, p, layer)
            if not any(dead[v] for v in r):
                continue
            cand = {v for v in r if not dead[v]}
            for v in r:
                if dead[v]:
                    cand.update(u for u in _row(g, v, layer) if not dead[u])
            cand.discard(p)
            repaired[(p, layer)] = _reselect(p, cand, dist, min(efc, len(cand)), M if layer else M0) if cand else []
    indeg_old = np.zeros(n, np.int64)
    for p in range(n):
        for v in _row(g, p, 0):
            indeg_old[v] += 1
    # 3. entry point
    entry = int(g["entry"])
    if dead[entry]:
        entry = int(live[np.argmax(levels[live])]) if len(live) else 0
    # 4. renumbering: new id = live ids below the old id
    remap = np.full(n, INV, np.int64)
    remap[live] = np.arange(len(live))
    nn = len(live)
    out = {
        "vectors": np.asarray(g["vectors"])[live],
        "labels": np.asarray(g["labels"])[live],
        "levels": np.asarray(g["levels"])[live],
        "links0": np.full((nn, M0), INV, np.uint32),
        "up_off": np.full(nn, INV, np.uint32),
    }
    up = []
    for i, p in enumerate(live.tolist()):
        for layer in range(levels[p] + 1):
            r = repaired.get((p, layer), _row(g, p, layer))
            row = np.full(M0 if layer == 0 else M, INV, np.uint32)
            row[:len(r)] = remap[np.asarray(r, np.int64)]
            if layer == 0:
                out["links0"][i] = row
            else:
                if layer == 1:
                    out["up_off"][i] = len(up)
                up.append(row)
    out["links_up"] = np.asarray(up, np.uint32).reshape(-1, M)
    out["entry"] = int(remap[entry]) if nn else 0
    out["maxlevel"] = int(levels[entry]) if nn else -1
    # 5. orphans: an empty level-0 row, or level-0 in-links before and none after
    indeg_new = np.zeros(nn, np.int64)
    for r in out["links0"]:
        for v in r[r != INV]:
            indeg_new[v] += 1
    empty = out["links0"][:, 0] == INV if nn else np.zeros(0, bool)
    orphans = np.flatnonzero(empty | ((indeg_old[live] > 0) & (indeg_new == 0)))
    return out, orphans


def compact_oracle(o, dead_labels, dist, efc=200):
    """OracleHNSW -> a new OracleHNSW holding the compacted index (orphans re-linked by updatePoint, in ascending
    new id).  dist(i, ids) works on the *pre-compaction* internal ids of `o`.  Returns (oracle, graph before the
    re-linking, orphans)."""
    g = o.export_graph()
    dead = np.isin(g["labels"], np.asarray(dead_labels, np.uint64))
    cg, orphans = compact_graph(g, dead, dist, o.M, efc)
    nn = len(cg["labels"])
    c = orc.OracleHNSW(o.dim, o.metric, max(nn, 1), M=o.M, ef_construction=efc)
    if nn:
        c.import_graph(cg)
    for i in orphans.tolist():
        c.add(cg["vectors"][i:i + 1], cg["labels"][i:i + 1], threads=1)
    return c, cg, orphans


def float_dist(x, metric):
    """dist(i, ids) over fp32 rows (as the oracle stores them: normalised for cosine)."""
    x = np.asarray(x, np.float32)
    if metric == "l2":
        return lambda i, ids: ((x[ids] - x[i]) ** 2).sum(1)
    return lambda i, ids: 1.0 - x[ids] @ x[i]


def int_ip_dist(x):
    """Exact 1 - dot over int64 rows (tie-free integer data)."""
    x = np.asarray(x, np.int64)
    return lambda i, ids: (1 - x[ids] @ x[i]).astype(np.float64)
