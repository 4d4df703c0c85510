"""CPU model of the fp32 walk's screen: what share of screened candidates each screen bound lets through.

Builds an oracle HNSW graph (M = 16, ef_construction = 200) over the first N rows of the benchmark's Gaussian stream
(seed 1234, inner product), re-walks Q queries (seed 4321) with hnswlib's searchKnn / searchBaseLayerST in numpy, and
for every evaluation made at a base-layer hop that started with a full result set (the evaluations the walk
screens) records the fp32 inner product, the hop-start worst distance, and whether each bound keeps the candidate:
  bf16:  L = 1 - E_b - (c S + A),       E_b = q . RN_bf16(x),  S = sum |q| |RN_bf16(x)|,  c = bf16 screen constant
  int8:  L = 1 - s E_c - (g |q|_2 (2 |x|_2 + |r|_2) + min(|q|_1 max|r|, |q|_2 |r|_2) + A),
         E_c = q . c,  c = RN(x / s) with s = max|x| / 127,  r = x - s c,  g = dpad 2^-24 / (1 - dpad 2^-24)
A candidate is kept when L < worst.  The fp32 rounding of the chains is not modelled (it moves L by far less than
the bounds).  Prints one JSON line: evaluations per query, the screened share, each screen's survivor share, and
the projected algorithmic bytes per query of the row reads (dim bytes + 16 bytes of per-row terms per int8-screened
evaluation, 2 dim per bf16-screened one, 4 dim per fp32 row read).  It also reports the share of screened hops whose
next node the int8 bounds prove: spec, the closest unexpanded result before the hop's candidates, is expanded next
when every int8 survivor has L > dist(spec) (no survivor can then come before it or evict it).  For the upper-layer
greedy descent, which the walk screens against the current node's distance, it reports the evaluations per query,
the share of them that survive the int8 bound (L < current distance) and the hops that move the descent, and the
projected row bytes per query with the descent read in fp32 and with it screened.

  python tools/walk_screen_int8_survival.py [--n 200000] [--dim 768] [--queries 300] [--ef 128] [--threads 8]
"""
import argparse
import heapq
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def bench_rows(n, d, seed=1234, chunk=1 << 20):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.standard_normal((min(chunk, n - i), d), dtype=np.float32) for i in range(0, n, chunk)])


def to_bf16(x):
    u = x.view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32).view(np.float32)


def bf16_constant(n):
    u, e = 1.0 / 256.0, n * 2.0 ** -24
    g = e / (1.0 - e)
    return (u + (2.0 + u) * g) / (1.0 - g)


def int8_copy(x):
    """per-row scale, codes, and the residual terms (max |r|, |r|_2) and |x|_2, in float64"""
    xd = x.astype(np.float64)
    s = np.abs(xd).max(1) / 127.0
    s = s.astype(np.float32).astype(np.float64)
    safe = np.where(s > 0, s, 1.0)
    c = np.clip(np.rint(xd / safe[:, None]), -127, 127)
    r = xd - s[:, None] * c
    return s, c.astype(np.float32), np.abs(r).max(1), np.linalg.norm(r, axis=1), np.linalg.norm(xd, axis=1)


def walk(g, x, q, ef, visit, visit_up):
    """hnswlib searchKnn (no deletions) under 1 - dot; visit(worst or None, spec, ids, dists) sees each base-layer
    hop's new candidates with the hop-start worst distance when the result set was full, and the distance of the
    closest unexpanded result at the hop's start (None when there is none); visit_up(cur_dist, ids, dists) sees each
    upper-layer descent hop's neighbours with the current node's distance"""
    links0, up_off, links_up = g["links0"], g["up_off"], g["links_up"]
    dist = lambda ids: 1.0 - x[ids] @ q
    cur = int(g["entry"])
    cd = float(dist(np.array([cur]))[0])
    for level in range(int(g["maxlevel"]), 0, -1):
        changed = True
        while changed:
            changed = False
            row = links_up[up_off[cur] + level - 1]
            ids = row[row != 0xFFFFFFFF]
            if len(ids):
                ds = dist(ids)
                visit_up(cd, ids, ds)
                j = int(np.argmin(ds))
                if ds[j] < cd:
                    cd, cur, changed = float(ds[j]), int(ids[j]), True
    visited = {cur}
    top = [(-cd, cur)]            # max-heap of results
    cand = [(cd, cur)]            # min-heap of candidates
    lower = cd
    while cand:
        d0, node = heapq.heappop(cand)
        if d0 > lower and len(top) == ef:
            break
        row = links0[node]
        ids = np.array([i for i in row[row != 0xFFFFFFFF] if i not in visited], dtype=np.int64)
        if not len(ids):
            continue
        visited.update(ids.tolist())
        ds = dist(ids)
        spec = cand[0][0] if cand and cand[0][0] <= lower else None  # an entry beyond lower was evicted
        visit(lower if len(top) == ef else None, spec, ids, ds)
        for i, dd in zip(ids.tolist(), ds.tolist()):
            if len(top) < ef or lower > dd:
                heapq.heappush(cand, (dd, i))
                heapq.heappush(top, (-dd, i))
                if len(top) > ef:
                    heapq.heappop(top)
                lower = -top[0][0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--queries", type=int, default=300)
    ap.add_argument("--ef", type=int, default=128)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    a = ap.parse_args()
    from oracle.oracle import OracleHNSW

    d = a.dim
    dpad = next(p for p in (384, 512, 768, 1024, 1536, 2048) if d <= p)
    t0 = time.time()
    x = bench_rows(a.n, d)
    o = OracleHNSW(d, "ip", max_elements=a.n, M=16, ef_construction=200)
    o.add(x, threads=a.threads)
    g = o.export_graph()
    x = g["vectors"]
    build_s = time.time() - t0
    b = to_bf16(x)
    s, c, rinf, r2, nx = int8_copy(x)
    gam = dpad * 2.0 ** -24 / (1 - dpad * 2.0 ** -24)
    cb = bf16_constant(dpad)
    qs = np.random.default_rng(4321).standard_normal((a.queries, d), dtype=np.float32)
    tot = {"evals": 0, "screened": 0, "bf16_kept": 0, "int8_kept": 0, "admissible": 0, "hops": 0, "proven": 0,
           "up_evals": 0, "up_kept": 0, "up_moves": 0}
    margins = {"bf16": [], "int8": []}
    for q in qs:
        qd = q.astype(np.float64)
        q1, q2 = np.abs(qd).sum(), np.linalg.norm(qd)
        A = dpad * (2.0 ** -125 * np.abs(qd).max() + 2.0 ** -124)

        def int8_lower(ids):
            mi = gam * q2 * (2 * nx[ids] + r2[ids]) + np.minimum(q1 * rinf[ids], q2 * r2[ids]) + A
            return 1.0 - s[ids] * (c[ids].astype(np.float64) @ qd) - mi, mi

        def visit_up(cd, ids, ds):
            tot["up_evals"] += len(ids)
            tot["up_kept"] += int((int8_lower(ids)[0] < cd).sum())
            tot["up_moves"] += int(ds.min() < cd)

        def visit(worst, spec, ids, ds):
            tot["evals"] += len(ids)
            if worst is None:
                return
            tot["screened"] += len(ids)
            mb = cb * (np.abs(b[ids]).astype(np.float64) @ np.abs(qd)) + A
            lb = 1.0 - b[ids].astype(np.float64) @ qd - mb
            li, mi = int8_lower(ids)
            tot["bf16_kept"] += int((lb < worst).sum())
            tot["int8_kept"] += int((li < worst).sum())
            tot["admissible"] += int((ds < worst).sum())
            tot["hops"] += 1
            tot["proven"] += int(spec is not None and bool(np.all(li[li < worst] > spec)))
            margins["bf16"].append(mb)
            margins["int8"].append(mi)

        walk(g, x, q, a.ef, visit, visit_up)
    nq = a.queries
    ue, uk = tot["up_evals"] / nq, tot["up_kept"] / max(tot["up_evals"], 1)
    ev, sc = tot["evals"] / nq, tot["screened"] / nq
    kb, ki = tot["bf16_kept"] / max(tot["screened"], 1), tot["int8_kept"] / max(tot["screened"], 1)
    unscreened = ev - sc
    bytes_bf16 = unscreened * 4 * d + sc * 2 * d + sc * kb * 4 * d
    bytes_int8 = unscreened * 4 * d + sc * (d + 16) + sc * ki * 4 * d
    # with the descent's rows: read in fp32, or screened (int8 rows and terms, fp32 rows of the survivors)
    bytes_descent_fp32 = bytes_int8 + ue * 4 * d
    bytes_descent_int8 = bytes_int8 + ue * (d + 16) + ue * uk * 4 * d
    print(json.dumps({
        "n": a.n, "dim": d, "dpad": dpad, "queries": nq, "ef": a.ef, "graph_build_s": round(build_s, 1),
        "evals_per_query": round(ev, 1), "screened_share": round(sc / ev, 4),
        "admissible_share": round(tot["admissible"] / max(tot["screened"], 1), 4),
        "bf16_survivor_share": round(kb, 4), "int8_survivor_share": round(ki, 4),
        "bf16_margin_median": round(float(np.median(np.concatenate(margins["bf16"]))), 3),
        "int8_margin_median": round(float(np.median(np.concatenate(margins["int8"]))), 3),
        "fp32_rows_per_eval_bf16": round((unscreened + sc * kb) / ev, 4),
        "fp32_rows_per_eval_int8": round((unscreened + sc * ki) / ev, 4),
        "row_bytes_per_query_bf16": round(bytes_bf16), "row_bytes_per_query_int8": round(bytes_int8),
        "row_bytes_ratio": round(bytes_int8 / bytes_bf16, 4),
        "int8_proven_next_share": round(tot["proven"] / max(tot["hops"], 1), 4),
        "descent_evals_per_query": round(ue, 1), "descent_int8_survivor_share": round(uk, 4),
        "descent_moves_per_query": round(tot["up_moves"] / nq, 2),
        "row_bytes_per_query_with_descent_fp32": round(bytes_descent_fp32),
        "row_bytes_per_query_with_descent_int8": round(bytes_descent_int8),
        "descent_screen_bytes_ratio": round(bytes_descent_int8 / bytes_descent_fp32, 4)}))


if __name__ == "__main__":
    main()
