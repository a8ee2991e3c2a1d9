"""NumPy ORACLE for path (iii) — TEST INFRASTRUCTURE ONLY.

Restates modules/finding/similarity.py:11-83 (sim, csls_sim, calculate_nearest_k),
modules/finding/alignment.py:13-84,146-168 (greedy_alignment, calculate_rank),
modules/bootstrapping/alignment_finder.py:28-76 (find_alignment = threshold ∧ row top-k) and
modules/train/batch.py:157-165 (find_neighbours) with ONE deliberate clarification: ties are broken
"lower column index first" (the reference's argsort/argpartition tie order is unspecified).
Pinned against the reference's own functions by tests/test_oracle_finding.py and tests/golden/*.npz.
"""
import numpy as np


def normalize_rows(x):
    """sklearn.preprocessing.normalize (similarity.py:30-32) as scikit-learn >= 1.0 does it: unit L2 rows; a row whose
    float32 norm is below 10·eps (a zero row, or one whose squared norm underflows) is left unchanged."""
    x = np.asarray(x, dtype=np.float32)
    n = np.sqrt((x.astype(np.float32) ** 2).sum(1, keepdims=True))
    n[n < 10 * np.finfo(np.float32).eps] = 1.0
    return (x / n).astype(np.float32)


def sim(e1, e2, metric="inner", normalize=False, csls_k=0):
    """similarity.py:11-54.  float32 result.  manhattan/euclidean/cosine go through float64 as cdist does."""
    e1 = np.asarray(e1, dtype=np.float32)
    e2 = np.asarray(e2, dtype=np.float32)
    if normalize:
        e1, e2 = normalize_rows(e1), normalize_rows(e2)
    if metric == "inner" or (metric == "cosine" and normalize):
        s = np.matmul(e1, e2.T)
    elif metric == "euclidean":
        a, b = e1.astype(np.float64), e2.astype(np.float64)
        d2 = (a * a).sum(1)[:, None] - 2 * a @ b.T + (b * b).sum(1)[None, :]
        s = (1 - np.sqrt(np.maximum(d2, 0))).astype(np.float32)
    elif metric == "cosine":
        a, b = normalize_rows(e1).astype(np.float64), normalize_rows(e2).astype(np.float64)
        s = (a @ b.T).astype(np.float32)   # 1 − (1 − cos)
    elif metric == "manhattan":
        a, b = e1.astype(np.float64), e2.astype(np.float64)
        s = np.empty((a.shape[0], b.shape[0]), dtype=np.float32)
        for i in range(a.shape[0]):
            s[i] = (1 - np.abs(a[i][None, :] - b).sum(1)).astype(np.float32)
    else:
        raise ValueError(metric)
    if csls_k > 0:
        s = csls_sim(s, csls_k)
    return s


def nearest_k_mean(s, k):
    """calculate_nearest_k (similarity.py:80-83): mean of the k largest of every row (true top-k mean)."""
    part = -np.partition(-s, k - 1, axis=1)[:, :k]
    return part.mean(axis=1, dtype=np.float32).astype(np.float32)


def csls_sim(s, k):
    """csls_sim (similarity.py:57-77): 2·S − r_i − c_j in float32, same operation order."""
    r = nearest_k_mean(s, k)
    c = nearest_k_mean(s.T, k)
    out = 2 * s.T - r
    return (out.T - c).astype(np.float32)


def rank_rows(s, gold=None):
    """calculate_rank (alignment.py:146-168) semantics per row: (argmax, 0-based rank of gold), ties → lower index."""
    n = s.shape[0]
    gold = np.arange(n) if gold is None else np.asarray(gold)
    g = s[np.arange(n), gold]
    better = (s > g[:, None]).sum(1)
    cols = np.arange(s.shape[1])[None, :]
    ties_before = ((s == g[:, None]) & (cols < gold[:, None])).sum(1)
    return s.argmax(1).astype(np.int32), (better + ties_before).astype(np.int32)


def metrics_from_ranks(rank, top_k):
    """Hits@k (% rounded to 3 dp), MR, MRR as alignment.py:60-67,160-167."""
    n = len(rank)
    hits = [round(float((rank < k).sum()) / n * 100, 3) for k in top_k]
    mr = float((rank + 1).sum() / n)
    mrr = float((1.0 / (rank + 1)).sum() / n)
    return hits, mr, mrr


def greedy_alignment(e1, e2, top_k, metric, normalize, csls_k):
    """greedy_alignment(accurate=True) (alignment.py:13-84) → (pairs set, hits list, mr, mrr)."""
    s = sim(e1, e2, metric, normalize, csls_k)
    top1, rank = rank_rows(s)
    hits, mr, mrr = metrics_from_ranks(rank, top_k)
    return {(i, int(j)) for i, j in enumerate(top1)}, hits, mr, mrr


def greedy_alignment_mt(e1, e2, top_k, metric, normalize, csls_k, nums_threads):
    """greedy_alignment with the reference's task split (alignment.py:43-60: rows divided into `nums_threads` tasks, one
    worker each, partial results merged); workers are threads here (the NumPy kernels release the GIL) instead of a
    multiprocessing pool that pickles its slice of the matrix.  Same results as greedy_alignment."""
    from concurrent.futures import ThreadPoolExecutor
    s = sim(e1, e2, metric, normalize, csls_k)
    n = s.shape[0]
    bounds = np.linspace(0, n, max(1, int(nums_threads)) + 1).astype(int)
    tasks = [(int(a), int(b)) for a, b in zip(bounds[:-1], bounds[1:]) if b > a]
    with ThreadPoolExecutor(max_workers=len(tasks)) as pool:
        parts = list(pool.map(lambda ab: rank_rows(s[ab[0]:ab[1]], np.arange(ab[0], ab[1])), tasks))
    top1 = np.concatenate([p[0] for p in parts])
    rank = np.concatenate([p[1] for p in parts])
    hits, mr, mrr = metrics_from_ranks(rank, top_k)
    return {(i, int(j)) for i, j in enumerate(top1)}, hits, mr, mrr


def topk_rows(s, k):
    """Per-row k largest (values, indices), sorted descending, ties → lower index."""
    order = np.lexsort((np.broadcast_to(np.arange(s.shape[1]), s.shape), -s), axis=1)[:, :k]
    return np.take_along_axis(s, order, 1), order.astype(np.int32)


def find_alignment(s, sim_th, k):
    """alignment_finder.py:28-51: {(i,j): s_ij > th} ∩ {(i,j): j among the k nearest of row i}; None if empty."""
    vals, idx = topk_rows(s, k) if k > 0 else (None, None)
    if k <= 0:
        x, y = np.where(s > sim_th)
        pairs = set(zip(x.tolist(), y.tolist()))
    else:
        pairs = {(i, int(idx[i, m])) for i in range(s.shape[0]) for m in range(k) if vals[i, m] > sim_th}
    return pairs if pairs else None


def find_neighbours(sub_embed, embed, entity_list, k):
    """batch.py:157-165: per row the SET of the k most similar (inner product) entities."""
    s = np.matmul(np.asarray(sub_embed, np.float32), np.asarray(embed, np.float32).T)
    _, idx = topk_rows(s, k)
    ent = np.asarray(entity_list)
    return [set(ent[row].tolist()) for row in idx]
