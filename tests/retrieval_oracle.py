"""The instance retrieval protocol (dinov3_jax/eval/retrieval.py) stated in float64 on the CPU: the full ranking by
descending similarity with ties to the lower index, the revisited Easy / Medium / Hard ground truth, the junk-free
ranks, the trapezoid AP and mP@k."""
import numpy as np

PROTOCOLS = ("easy", "medium", "hard")
KS = (1, 5, 10)


def ok_junk(easy, hard, junk, protocol):
    """(ok, junk) index sets of one query under a protocol; an index in both counts as ok."""
    easy, hard, junk = (set(int(v) for v in np.asarray(l).reshape(-1)) for l in (easy, hard, junk))
    ok, jk = {"easy": (easy, junk | hard), "medium": (easy | hard, junk), "hard": (hard, junk | easy)}[protocol]
    return ok, jk - ok


def order(sim_row):
    """Database indices by descending similarity, ties to the lower index."""
    s = np.asarray(sim_row, np.float64)
    return np.lexsort((np.arange(len(s)), -s))


def ranks(sim_row):
    """int [N]: the 0-based rank of every database index."""
    o = order(sim_row)
    r = np.empty(len(o), np.int64)
    r[o] = np.arange(len(o))
    return r


def junk_free_ranks(rank, ok, junk):
    """The sorted 0-based ranks of the ok images, each reduced by the junk images ranked above it."""
    pos = np.sort([rank[i] for i in ok]).astype(np.int64)
    jr = np.sort([rank[i] for i in junk]).astype(np.int64)
    return pos - np.searchsorted(jr, pos)


def average_precision(r):
    """The revisited trapezoid over sorted junk-free 0-based ranks r; NaN when there are none."""
    if len(r) == 0:
        return float("nan")
    ap = 0.0
    for j, rj in enumerate(r):
        ap += (1.0 if rj == 0 else j / rj) + (j + 1) / (rj + 1)
    return ap / (2.0 * len(r))


def precision_at(r, k):
    """P@k over sorted junk-free 0-based ranks r: 1-based ranks, kq = min(max rank, k), |{rank <= kq}| / kq."""
    if len(r) == 0:
        return float("nan")
    pos = np.asarray(r) + 1
    kq = min(int(pos.max()), k)
    return float((pos <= kq).sum()) / kq


def query_scores(sim_row, easy, hard, junk):
    """{protocol: (AP, [P@1, P@5, P@10], n_ok)} of one query."""
    rank = ranks(sim_row)
    out = {}
    for p in PROTOCOLS:
        ok, jk = ok_junk(easy, hard, junk, p)
        r = junk_free_ranks(rank, ok, jk)
        out[p] = (average_precision(r), [precision_at(r, k) for k in KS], len(ok))
    return out


def evaluate(sim, easy, hard, junk):
    """{"mAP": {protocol}, "mP@k": {protocol: {"1", "5", "10"}}, "n_empty": {protocol}} in percent over the queries
    with ok images, and the per-query scores."""
    per = [query_scores(sim[q], easy[q], hard[q], junk[q]) for q in range(len(sim))]
    res = {"mAP": {}, "mP@k": {}, "n_empty": {}}
    for p in PROTOCOLS:
        keep = [s[p] for s in per if s[p][2] > 0]
        res["n_empty"][p] = len(per) - len(keep)
        res["mAP"][p] = 100.0 * float(np.mean([s[0] for s in keep])) if keep else float("nan")
        res["mP@k"][p] = {str(k): (100.0 * float(np.mean([s[1][t] for s in keep])) if keep else float("nan"))
                          for t, k in enumerate(KS)}
    return res, per
