"""numpy reference of the batched top-k contract (include/kge_b200.h, kge_topk_*): eligible candidates ordered by
(NaN last, score with -0 == +0, smaller id first); fewer than k left -> id -1, score NaN."""
import numpy as np

NAN_BITS = 0x7FC00000


def ref_topk(scores, k, descending=False, filt=None):
    """one row -> (ids [k] int64, score bits [k] uint32)"""
    scores = np.ascontiguousarray(scores, dtype=np.float32)
    n = len(scores)
    elig = np.ones(n, dtype=bool)
    if filt is not None and len(filt):
        f = np.asarray(filt, dtype=np.int64)
        elig[f[(f >= 0) & (f < n)]] = False
    ids = np.flatnonzero(elig)
    s = scores[ids].astype(np.float64)
    nan = np.isnan(s)
    s = np.where(nan, 0.0, -s if descending else s) + 0.0   # + 0.0 folds -0 onto +0
    top = ids[np.lexsort((ids, s, nan))][:k]
    out_ids = np.full(k, -1, dtype=np.int64)
    out_bits = np.full(k, NAN_BITS, dtype=np.uint32)
    out_ids[:len(top)] = top
    out_bits[:len(top)] = scores[top].view(np.uint32)
    return out_ids, out_bits


def csr(rows):
    """list of per-query id lists -> (ptr [Q+1], idx [nnz]) int64"""
    ptr = np.zeros(len(rows) + 1, dtype=np.int64)
    ptr[1:] = np.cumsum([len(r) for r in rows])
    idx = np.concatenate([np.asarray(r, dtype=np.int64) for r in rows] + [np.zeros(0, np.int64)])
    return ptr, idx
