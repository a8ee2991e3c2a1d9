"""Host side of path (iii): similarity / CSLS / top-k / rank / neighbour search through liboea.so.

Mirrors the call signatures of the reference's modules/finding/{similarity,alignment}.py and
modules/train/batch.py:145-165 but keeps everything on the device; inputs may be NumPy arrays (reference
API) or CUDA tensors (internal fast path: no host round trip).  No fallback to NumPy/torch maths.
"""
import ctypes as C
import time

import collections.abc

import numpy as np
import torch

from . import lib as L
from .engine import _ptr, _stream_ptr, pitch_for

_METRICS = {"inner": L.METRIC_INNER, "cosine": L.METRIC_INNER, "euclidean": L.METRIC_L2, "manhattan": L.METRIC_L1}


def _device():
    if not torch.cuda.is_available():
        raise L.OeaError("openea_b200.finding needs a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def to_device_rows(x, normalize=False):
    """→ float32 CUDA tensor [n, pitch] with zero padding (pitch % 4 == 0); optional sklearn-style row normalise."""
    lib = L.load()
    dev = _device()
    t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=np.float32)))
    t = t.to(device=dev, dtype=torch.float32)
    n, d = t.shape
    p = pitch_for(d)
    if not normalize and p == d and t.is_contiguous():
        return t, d
    out = torch.zeros(n, p, dtype=torch.float32, device=dev)
    if normalize:
        t = t.contiguous()
        L.check(lib.oea_rows_normalize(_ptr(t), d, n, d, _ptr(out), p, _stream_ptr()), "oea_rows_normalize")
    else:
        out[:, :d] = t
    return out, d


def kmajor(t, tc=None):
    """k-major zero-padded copy of prepared rows [n, pitch] (oea_sim_transpose) → (tensor, ld).  `tc` is a per-call
    cache {id(tensor): result} so that the passes of one evaluation share the copies (never cached across calls:
    the caller may change the rows in place)."""
    if tc is not None and id(t) in tc:
        return tc[id(t)][1:]
    lib = L.load()
    n, pitch = t.shape
    ld = lib.oea_sim_transpose_ld(n)
    out = torch.empty(lib.oea_sim_transpose_bytes(n, pitch) // 4, dtype=torch.float32, device=t.device)
    L.check(lib.oea_sim_transpose(_ptr(t), pitch, n, _ptr(out), _stream_ptr()), "oea_sim_transpose")
    if tc is not None:
        tc[id(t)] = (t, out, ld)      # keeps `t` alive so the id stays unique for the duration of the call
    return out, ld


def _cfg(metric, e1, e2, d, tc=None):
    if metric not in _METRICS:
        raise ValueError("metric %r is not supported by the CUDA engine (inner/cosine/euclidean/manhattan)" % (metric,))
    assert e1.is_contiguous() and e2.is_contiguous()
    t1, ld1 = kmajor(e1, tc)
    t2, ld2 = kmajor(e2, tc) if e2 is not e1 else (t1, ld1)
    cfg = L.SimCfg(_METRICS[metric], e1.shape[0], e2.shape[0], d, e1.shape[1], e2.shape[1], t1.data_ptr(), t2.data_ptr(),
                   ld1, ld2)
    cfg._keep = (t1, t2)              # the k-major copies must outlive the (asynchronous) kernels using them
    return cfg


def _prep_pair(embed1, embed2, metric, normalize):
    # 'cosine' without normalize is 1 − cosine distance = cosine similarity: normalise, then inner product
    norm = bool(normalize) or metric == "cosine"
    e1, d = to_device_rows(embed1, norm)
    e2, d2 = to_device_rows(embed2, norm)
    assert d == d2, "embedding dimensions differ"
    return e1, e2, d


def topk(e1, e2, d, metric, k, row_off=None, col_off=None, want=("val", "idx", "mean"), tc=None):
    """Per-row top-k of S (or CSLS S' when offsets are given) of prepared device rows → dict of tensors."""
    lib = L.load()
    cfg = _cfg(metric, e1, e2, d, tc)
    n1 = e1.shape[0]
    dev = e1.device
    ws_bytes = lib.oea_sim_topk_workspace_bytes(C.byref(cfg), k)
    ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)
    out = {}
    val = torch.empty(n1, k, dtype=torch.float32, device=dev) if "val" in want else None
    idx = torch.empty(n1, k, dtype=torch.int32, device=dev) if "idx" in want else None
    mean = torch.empty(n1, dtype=torch.float32, device=dev) if "mean" in want else None
    L.check(lib.oea_sim_topk(C.byref(cfg), _ptr(e1), _ptr(e2), _ptr(row_off), _ptr(col_off), k,
                             _ptr(val), _ptr(idx), _ptr(mean), _ptr(ws), ws_bytes, _stream_ptr()), "oea_sim_topk")
    out["val"], out["idx"], out["mean"] = val, idx, mean
    return out


def csls_offsets(e1, e2, d, metric, k, tc=None):
    """r_i = mean of the k nearest of row i, c_j = mean of the k nearest of column j (similarity.py:73-83)."""
    tc = {} if tc is None else tc
    r = topk(e1, e2, d, metric, k, want=("mean",), tc=tc)["mean"]
    c = topk(e2, e1, d, metric, k, want=("mean",), tc=tc)["mean"]
    return r, c


def rank(e1, e2, d, metric, gold, row_off=None, col_off=None, tc=None):
    """(argmax column, 0-based rank of gold[i]) per row → two int32 CUDA tensors."""
    lib = L.load()
    cfg = _cfg(metric, e1, e2, d, tc)
    n1, dev = e1.shape[0], e1.device
    gold_t = torch.as_tensor(gold, dtype=torch.int32, device=dev).contiguous()
    ws_bytes = lib.oea_sim_rank_workspace_bytes(C.byref(cfg))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    top1 = torch.empty(n1, dtype=torch.int32, device=dev)
    rk = torch.empty(n1, dtype=torch.int32, device=dev)
    L.check(lib.oea_sim_rank(C.byref(cfg), _ptr(e1), _ptr(e2), _ptr(row_off), _ptr(col_off), _ptr(gold_t),
                             _ptr(top1), _ptr(rk), _ptr(ws), ws_bytes, _stream_ptr()), "oea_sim_rank")
    return top1, rk


def sim_matrix(e1, e2, d, metric, row_off=None, col_off=None, out=None, tc=None):
    lib = L.load()
    cfg = _cfg(metric, e1, e2, d, tc)
    if out is None:
        out = torch.empty(e1.shape[0], e2.shape[0], dtype=torch.float32, device=e1.device)
    L.check(lib.oea_sim_matrix(C.byref(cfg), _ptr(e1), _ptr(e2), _ptr(row_off), _ptr(col_off), _ptr(out),
                               out.stride(0), _stream_ptr()), "oea_sim_matrix")
    return out


def sim(embed1, embed2, metric="inner", normalize=False, csls_k=0):
    """Drop-in for modules/finding/similarity.py:11 `sim` → float32 CUDA tensor [n1, n2]."""
    e1, e2, d = _prep_pair(embed1, embed2, metric, normalize)
    r = c = None
    tc = {}
    if csls_k > 0:
        r, c = csls_offsets(e1, e2, d, metric, csls_k, tc)
    return sim_matrix(e1, e2, d, metric, r, c, tc=tc)


MATERIALIZE_MAX_BYTES = 48 << 30   # CSLS runs on a stored n1×n2 matrix (1 contraction pass) below this size


def use_tensor_cores(metric):
    """OEA_SIM_TC=1 routes the stored similarity matrix of the materialised evaluation through the 3xTF32 wgmma kernel
    (oea_sim_matrix_tc; inner / normalised-cosine only).  Off by default: its values equal the FP32 kernel's only to fp32
    round-off, so arg-max / rank may differ on exact near-ties (tests/test_sim_tc_gpu.py bounds how many)."""
    import os
    return os.environ.get("OEA_SIM_TC") == "1" and _METRICS[metric] == L.METRIC_INNER


def sim_matrix_tc(e1, e2, d, metric, row_off=None, col_off=None, out=None):
    """oea_sim_matrix_tc on prepared device rows → [n1, ld] tensor (ld = n2 rounded up to a multiple of 4)."""
    lib = L.load()
    cfg = _cfg(metric, e1, e2, d)
    n1, n2 = e1.shape[0], e2.shape[0]
    if out is None:
        out = torch.empty(n1, (n2 + 3) // 4 * 4, dtype=torch.float32, device=e1.device)
    L.check(lib.oea_sim_matrix_tc(C.byref(cfg), _ptr(e1), _ptr(e2), _ptr(row_off), _ptr(col_off), _ptr(out), out.stride(0),
                                  _stream_ptr()), "oea_sim_matrix_tc")
    return out


def _eval_materialized(e1, e2, d, metric, csls_k, gold):
    """CSLS evaluation with ONE contraction pass: S stored once (tile kernel, store epilogue), then three
    HBM-bound streaming kernels (row k-means, column k-means, rank)."""
    lib = L.load()
    n1, n2 = e1.shape[0], e2.shape[0]
    ld = (n2 + 3) // 4 * 4
    s = torch.empty(n1, ld, dtype=torch.float32, device=e1.device)
    cfg = _cfg(metric, e1, e2, d)
    st = _stream_ptr()
    if use_tensor_cores(metric):
        L.check(lib.oea_sim_matrix_tc(C.byref(cfg), _ptr(e1), _ptr(e2), None, None, _ptr(s), ld, st), "oea_sim_matrix_tc")
    else:
        L.check(lib.oea_sim_matrix(C.byref(cfg), _ptr(e1), _ptr(e2), None, None, _ptr(s), ld, st), "oea_sim_matrix")
    r = torch.empty(n1, dtype=torch.float32, device=e1.device)
    c = torch.empty(n2, dtype=torch.float32, device=e1.device)
    L.check(lib.oea_matrix_topk_mean(_ptr(s), ld, n1, n2, csls_k, 0, _ptr(r), None, 0, st), "oea_matrix_topk_mean")
    ws_bytes = lib.oea_matrix_topk_mean_workspace_bytes(n1, n2, csls_k, 1)
    ws = torch.empty(max(16, ws_bytes), dtype=torch.uint8, device=e1.device)
    L.check(lib.oea_matrix_topk_mean(_ptr(s), ld, n1, n2, csls_k, 1, _ptr(c), _ptr(ws), ws_bytes, st),
            "oea_matrix_topk_mean")
    top1 = torch.empty(n1, dtype=torch.int32, device=e1.device)
    rk = torch.empty(n1, dtype=torch.int32, device=e1.device)
    L.check(lib.oea_matrix_rank(_ptr(s), ld, n1, n2, _ptr(r), _ptr(c), _ptr(gold), _ptr(top1), _ptr(rk), st),
            "oea_matrix_rank")
    return top1, rk


def eval_alignment(embed1, embed2, top_k, metric, normalize, csls_k, gold=None, materialize=None):
    """The numeric core of greedy_alignment: returns (top1 idx tensor, rank tensor, hits list, mr, mrr).
    With CSLS the similarity matrix is stored once when it fits MATERIALIZE_MAX_BYTES (1 contraction pass + 3
    streaming passes); otherwise, and without CSLS, nothing is materialised (tile kernel with fused epilogues)."""
    e1, e2, d = _prep_pair(embed1, embed2, metric, normalize)
    n1 = e1.shape[0]
    if gold is None:
        gold = torch.arange(n1, dtype=torch.int32, device=e1.device)   # alignment.py:153: gold of row i is i
    gold = torch.as_tensor(gold, dtype=torch.int32, device=e1.device).contiguous()
    if materialize is None:
        materialize = csls_k > 0 and 4 * n1 * e2.shape[0] <= MATERIALIZE_MAX_BYTES and csls_k <= min(n1, e2.shape[0])
    if materialize and csls_k > 0:
        top1, rk = _eval_materialized(e1, e2, d, metric, csls_k, gold)
    else:
        r = c = None
        tc = {}
        if csls_k > 0:
            r, c = csls_offsets(e1, e2, d, metric, csls_k, tc)
        top1, rk = rank(e1, e2, d, metric, gold, r, c, tc=tc)
    hits, mr, mrr = rank_stats(rk, top_k)
    return top1, rk, hits, mr, mrr


def rank_stats(rk, top_k):
    """Hits@k (percent, 3 dp as alignment.py:66-69), MR and MRR of a device rank vector: one kernel, one D2H copy."""
    lib = L.load()
    n = rk.shape[0]
    ks = [int(k) for k in top_k]
    hits, sums = [], None
    for lo in range(0, max(1, len(ks)), 8):          # the kernel takes up to 8 thresholds per launch
        chunk = ks[lo:lo + 8]
        arr = (C.c_int32 * max(1, len(chunk)))(*chunk)
        out = torch.empty(len(chunk) + 2, dtype=torch.float64, device=rk.device)
        L.check(lib.oea_rank_stats(_ptr(rk), n, arr, len(chunk), _ptr(out), _stream_ptr()), "oea_rank_stats")
        vals = out.tolist()
        hits += [round(v / n * 100, 3) for v in vals[:len(chunk)]]
        sums = vals[len(chunk):]
    return hits, float(sums[0] / n), float(sums[1] / n)


class PairSet(collections.abc.Set):
    """The alignment result {(i, top1[i])} as an immutable set view over the device result's host copy: a drop-in for the
    Python set modules/finding/alignment.py:13 returns (membership, iteration, len, ==, set algebra), built without the
    70 000-tuple Python loop in the evaluation's critical path — tuples are produced only when something iterates."""

    __slots__ = ("_top1",)

    def __init__(self, top1):
        self._top1 = np.asarray(top1)

    def __len__(self):
        return int(self._top1.shape[0])          # row indices are distinct, so the pairs are

    def __iter__(self):
        return iter(zip(range(len(self)), self._top1.tolist()))

    def __contains__(self, pair):
        try:
            i, j = pair
            return 0 <= i < len(self) and int(self._top1[i]) == j
        except (TypeError, ValueError):
            return False

    @classmethod
    def _from_iterable(cls, it):                 # set algebra (|, &, -, ^) yields ordinary sets
        return set(it)

    def __repr__(self):
        return "PairSet(%d pairs)" % len(self)


def greedy_alignment(embed1, embed2, top_k, nums_threads, metric, normalize, csls_k, accurate):
    """Drop-in for modules/finding/alignment.py:13.  `nums_threads` is accepted and ignored (one GPU pass).
    Quick mode (accurate=False) computes the same exact ranks; only the printed line differs."""
    t = time.time()
    from . import parallel as par
    if par.replicas_in_sync():
        # one process per GPU with identical embeddings on every rank: every rank ranks its block of embed1's rows (one all-gather of partial column top-k
        # lists for CSLS), the statistics are all-reduced and the arg-max column of every row is gathered
        n1 = embed1.shape[0]
        hits, mr, mrr, (_, _, top1, _) = eval_alignment_sharded(embed1, embed2, top_k, metric, normalize, csls_k)
        top1 = par.allgather_blocks(top1, n1)
    else:
        top1, _, hits, mr, mrr = eval_alignment(embed1, embed2, top_k, metric, normalize, csls_k)
    alignment_rest = PairSet(top1.cpu().numpy())
    hits_arr = np.array(hits)
    cost = time.time() - t
    if accurate:
        if csls_k > 0:
            print("accurate results with csls: csls={}, hits@{} = {}%, mr = {:.3f}, mrr = {:.6f}, time = {:.3f} s ".
                  format(csls_k, top_k, hits_arr, mr, mrr, cost))
        else:
            print("accurate results: hits@{} = {}%, mr = {:.3f}, mrr = {:.6f}, time = {:.3f} s ".
                  format(top_k, hits_arr, mr, mrr, cost))
    else:
        if csls_k > 0:
            print("quick results with csls: csls={}, hits@{} = {}%, time = {:.3f} s ".format(csls_k, top_k, hits_arr, cost))
        else:
            print("quick results: hits@{} = {}%, time = {:.3f} s ".format(top_k, hits_arr, cost))
    return alignment_rest, hits_arr[0], mr, mrr


def stable_matching(embed1, embed2, metric, normalize, csls_k, cut=100):
    """Gale–Shapley (suitor-proposing, at most `cut` rounds) on the device: K3's top-`cut` list of every row is the
    suitor's preference list, reviewers rank by the same similarities (oea_gale_shapley; alignment.py:87-133,171-224).
    Returns (match [n1] int32 device tensor: the column held by row i or −1, rounds run)."""
    lib = L.load()
    e1, e2, d = _prep_pair(embed1, embed2, metric, normalize)
    n1, n2 = e1.shape[0], e2.shape[0]
    r = c = None
    if csls_k > 0:
        r, c = csls_offsets(e1, e2, d, metric, csls_k)
    kk = max(1, min(int(cut), n2))
    if kk <= 32:                      # K3's fused sorted top-k (one warp holds a row's list)
        res = topk(e1, e2, d, metric, kk, r, c, want=("val", "idx"))
        idx, val = res["idx"].contiguous(), res["val"].contiguous()
    else:                             # longer lists: materialise S (or CSLS S'), radix-select the set, order it
        if kk > 128:
            raise ValueError("stable_matching: cut > 128 is not supported on the device path")
        ld = (n2 + 3) // 4 * 4
        s = torch.empty(n1, ld, dtype=torch.float32, device=e1.device)
        sim_matrix(e1, e2, d, metric, r, c, out=s)
        idx = torch.empty(n1, kk, dtype=torch.int32, device=e1.device)
        val = torch.empty(n1, kk, dtype=torch.float32, device=e1.device)
        L.check(lib.oea_rows_select_topk(_ptr(s), ld, n1, n2, kk, None, _ptr(idx), _stream_ptr()), "oea_rows_select_topk")
        L.check(lib.oea_rows_gather_sort(_ptr(s), ld, n1, kk, _ptr(idx), _ptr(val), _stream_ptr()), "oea_rows_gather_sort")
        del s
    match = torch.empty(n1, dtype=torch.int32, device=e1.device)
    ws_bytes = lib.oea_gale_shapley_workspace_bytes(n1, n2)
    ws = torch.empty(ws_bytes // 8 + 1, dtype=torch.int64, device=e1.device)
    rounds = C.c_int32(0)
    L.check(lib.oea_gale_shapley(_ptr(idx), _ptr(val), n1, n2, kk, int(cut), _ptr(match), _ptr(ws), ws.numel() * 8,
                                 C.byref(rounds), _stream_ptr()), "oea_gale_shapley")
    return match, int(rounds.value)


def find_neighbours_device(embeds, entity_list, k, row_block=8192):
    """ε-truncated neighbour search (batch.py:145-165) on device: for every row of `embeds` the k entities of
    `entity_list` with the largest inner product → int32 CUDA tensor [n, k] of ENTITY IDS (set semantics)."""
    lib = L.load()
    e, d = to_device_rows(embeds, False)
    n = e.shape[0]
    dev = e.device
    ids = torch.as_tensor(np.asarray(entity_list, dtype=np.int32) if not isinstance(entity_list, torch.Tensor) else entity_list,
                          dtype=torch.int32, device=dev).contiguous()
    assert ids.numel() == n
    out = torch.empty(n, k, dtype=torch.int32, device=dev)
    rb = min(n, row_block)
    ld = (n + 3) // 4 * 4
    buf = torch.empty(rb, ld, dtype=torch.float32, device=dev)
    tc = {}
    for r0 in range(0, n, rb):
        r1 = min(n, r0 + rb)
        sub = e[r0:r1]
        cfg = _cfg("inner", sub, e, d, tc)
        L.check(lib.oea_sim_matrix(C.byref(cfg), _ptr(sub), _ptr(e), None, None, _ptr(buf), ld, _stream_ptr()),
                "oea_sim_matrix")
        L.check(lib.oea_rows_select_topk(_ptr(buf), ld, r1 - r0, n, k, _ptr(ids), _ptr(out[r0:r1]), _stream_ptr()),
                "oea_rows_select_topk")
    return out


def find_alignment_device(embed1, embed2, sim_th, k, metric="inner", normalize=True):
    """Bootstrapping candidate pairs (alignment_finder.py:28-51): {(i,j): S_ij > th} ∩ {j in top-k of row i}.
    Returns (rows, cols, vals) CUDA tensors of the surviving pairs."""
    e1, e2, d = _prep_pair(embed1, embed2, metric, normalize)
    res = topk(e1, e2, d, metric, k, want=("val", "idx"))
    keep = res["val"] > sim_th
    rows = torch.arange(e1.shape[0], device=e1.device, dtype=torch.int32)[:, None].expand_as(keep)[keep]
    return rows, res["idx"][keep], res["val"][keep]


def eval_alignment_sharded(embed1, embed2, top_k, metric, normalize, csls_k):
    """Multi-GPU greedy_alignment core: this rank evaluates a contiguous block of embed1's rows against ALL of
    embed2 (replicated).  Row top-k / rank are local; the CSLS column means need one all-gather of each rank's
    partial [n2, k] column lists.  Returns (hits list, mr, mrr) of the WHOLE problem on every rank, plus this
    rank's (row range, top1, rank) tensors."""
    from . import parallel as par
    rank_id, ws = par.world()
    e1_all, e2, d = _prep_pair(embed1, embed2, metric, normalize)
    n1 = e1_all.shape[0]
    lo, hi = par.block_range(n1, rank_id, ws)
    e1 = e1_all[lo:hi].contiguous()
    r = c = None
    if csls_k > 0:
        tc = {}
        r = topk(e1, e2, d, metric, csls_k, want=("mean",), tc=tc)["mean"]             # local rows: exact
        part = topk(e2, e1, d, metric, min(csls_k, hi - lo), want=("val",), tc=tc)["val"]   # columns over MY rows
        if part.shape[1] < csls_k:   # fewer local rows than k: pad so the merge still sees k slots per rank
            pad = torch.full((part.shape[0], csls_k - part.shape[1]), -3.0e38, device=part.device)
            part = torch.cat([part, pad], 1)
        c = par.merge_partial_topk(par.allgather_partial(part), csls_k)
    gold = torch.arange(lo, hi, dtype=torch.int32, device=e1.device)
    top1, rk = rank(e1, e2, d, metric, gold, r, c)
    rk64 = rk.to(torch.float64)
    stats = torch.stack([(rk < k).sum().to(torch.float64) for k in top_k] + [(rk64 + 1).sum(), (1.0 / (rk64 + 1)).sum()])
    par.allreduce_sum(stats)
    stats = stats.cpu().numpy()
    hits = [round(float(x) / n1 * 100, 3) for x in stats[:len(top_k)]]
    return hits, float(stats[-2] / n1), float(stats[-1] / n1), (lo, hi, top1, rk)
