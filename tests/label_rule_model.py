"""numpy model of the key-mode self-removal of the reference's NearestNeighbor (server.cc:190-207,
offlinehub.py:110-130), as ehb_index_search_by_label_ex applies it to a k + 1 result list."""
import numpy as np

NO_LABEL = np.uint64(0xFFFFFFFFFFFFFFFF)


def drop_self(self_labels, labels, dists, counts, k):
    """[nq][k + 1] nearest-first results (counts hits each) -> [nq][k]: the own label is removed when present, else
    the last hit is dropped when there are k + 1; padded with NO_LABEL / +inf."""
    nq = len(self_labels)
    ol = np.full((nq, k), NO_LABEL, np.uint64)
    od = np.full((nq, k), np.inf, np.float32)
    oc = np.zeros(nq, np.uint32)
    for q in range(nq):
        c = int(counts[q])
        row_l, row_d = list(labels[q][:c]), list(dists[q][:c])
        hit = [j for j, l in enumerate(row_l) if l == self_labels[q]]
        if hit:
            del row_l[hit[0]], row_d[hit[0]]
        elif c > k:
            row_l, row_d = row_l[:k], row_d[:k]
        m = min(len(row_l), k)
        ol[q, :m], od[q, :m], oc[q] = row_l[:m], row_d[:m], m
    return ol, od, oc
