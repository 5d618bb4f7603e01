"""Row-range sharding of a FLAT corpus over ranks and the single exchange step of the KNN path.

One process per GPU (torchrun).  Each rank owns rows [lo, hi) of the corpus (labels travel with the
rows), scans its shard, and the per-shard top-k lists are exchanged with ONE all-gather and merged by
`(score asc, label asc)` — the coordinator merge of the reference (src/module.c:3139-3176, comparator
VS/utils/query_result_utils.h:19-23).  Exactness: the global top-k is a subset of the union of the local
top-k lists.  torch.distributed is plumbing only; the merge itself is a CUDA kernel
(VecSimB200_MergeShardTopK).

Posting lists shard by docId range with the same boundaries (SURVEY.md §8e): shard g owns docIds
(g*N/G, (g+1)*N/G]; every list is cut at the boundaries, each rank evaluates AND/OR + scorer + top-N on its slice
with the GLOBAL statistics, and the per-shard top-N lists are exchanged with one all-gather and merged by
`(score desc, docId asc)` (II_MergeShardTopN).
"""
import ctypes as C


def shard_range(n_total: int, world: int, rank: int):
    """Contiguous ranges; shard g owns rows [g*N/G, (g+1)*N/G) (SURVEY.md §8e)."""
    lo = (n_total * rank) // world
    hi = (n_total * (rank + 1)) // world
    return lo, hi


def allgather_topk(scores, labels, group=None):
    """scores [B,k] float32, labels [B,k] int64 (-1 = empty) on this rank -> ([G,B,k], [G,B,k])."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    gs = torch.empty((world,) + tuple(scores.shape), dtype=scores.dtype, device=scores.device)
    gl = torch.empty((world,) + tuple(labels.shape), dtype=labels.dtype, device=labels.device)
    if scores.is_cuda:
        dist.all_gather_into_tensor(gs, scores.contiguous(), group=group)
        dist.all_gather_into_tensor(gl, labels.contiguous(), group=group)
    else:  # gloo (CPU tests)
        ls = [torch.empty_like(scores) for _ in range(world)]
        ll = [torch.empty_like(labels) for _ in range(world)]
        dist.all_gather(ls, scores.contiguous(), group=group)
        dist.all_gather(ll, labels.contiguous(), group=group)
        gs, gl = torch.stack(ls), torch.stack(ll)
    return gs, gl


def merge_topk_device(gath_scores, gath_labels, stream_ptr=None):
    """[G,B,k] gathered lists on a CUDA device -> merged ([B,k], [B,k]) with the library's kernel."""
    import torch

    from . import vecsim

    G, B, k = gath_scores.shape
    out_s = torch.empty((B, k), dtype=torch.float32, device=gath_scores.device)
    out_l = torch.empty((B, k), dtype=torch.int64, device=gath_scores.device)
    sp = C.c_void_p(stream_ptr if stream_ptr is not None else torch.cuda.current_stream().cuda_stream)
    rc = vecsim.lib().VecSimB200_MergeShardTopK(gath_scores.data_ptr(), gath_labels.data_ptr(), G, B, k,
                                                out_s.data_ptr(), out_l.data_ptr(), sp)
    if rc != 0:
        raise RuntimeError("VecSimB200_MergeShardTopK failed")
    return out_s, out_l


def merge_shard_lists(parts, range_query=False, order=0, stream_ptr=None):
    """Per rank the (labels [nq,w] int64, scores [nq,w] float32, counts [nq] 32-bit) CUDA tensors of its local device call
    (HybridTopKBatchDevice, [Label|Hybrid]RangeQueryBatchDevice) -> the merged (labels, scores, counts) of all ranks.  Packs each
    rank's result into its counted exchange block (VecSimB200_ShardListBlockBytes), rank-major as an all-gather leaves them, and
    merges them with VecSimB200_MergeShardListBlocks on the device.  order: BY_SCORE (0) or BY_ID (1, range results only).
    Packing and merge run on `stream_ptr` (default: torch's current stream), so the local calls must be enqueued on that stream
    or be complete: a call left on another stream, e.g. the legacy default stream while torch's current stream is a non-blocking
    one, races with the packing."""
    import torch

    from . import vecsim

    L = vecsim.lib()
    nq, w = parts[0][0].shape
    dev = parts[0][0].device
    n = nq * w
    block = int(L.VecSimB200_ShardListBlockBytes(nq, w))
    blocks = torch.zeros((len(parts), block), dtype=torch.uint8, device=dev)
    for g, (labels, scores, counts) in enumerate(parts):
        blocks[g, :n * 8] = labels.contiguous().view(torch.uint8).reshape(-1)
        blocks[g, n * 8:n * 12] = scores.contiguous().view(torch.uint8).reshape(-1)
        blocks[g, n * 12:n * 12 + nq * 4] = counts.contiguous().view(torch.uint8).reshape(-1)
    out_l = torch.empty((nq, w), dtype=torch.int64, device=dev)
    out_s = torch.empty((nq, w), dtype=torch.float32, device=dev)
    out_c = torch.empty(nq, dtype=torch.int32, device=dev)
    sp = C.c_void_p(stream_ptr if stream_ptr is not None else torch.cuda.current_stream().cuda_stream)
    rc = L.VecSimB200_MergeShardListBlocks(blocks.data_ptr(), len(parts), nq, w, 1 if range_query else 0, order, out_l.data_ptr(),
                                           out_s.data_ptr(), out_c.data_ptr(), sp)
    if rc != 0:
        raise RuntimeError("VecSimB200_MergeShardListBlocks failed")
    return out_l, out_s, out_c


# ------------------------------------------------------------------------------------------------
# postings
# ------------------------------------------------------------------------------------------------
def doc_range(n_docs: int, world: int, rank: int):
    """docIds are 1..n_docs; shard g owns (lo, hi] with the row-shard boundaries."""
    return shard_range(n_docs, world, rank)


def split_posting_list(doc_ids, freqs, lo: int, hi: int):
    """Slice of an ascending docId array (and its freqs) inside (lo, hi] — binary search on the boundaries."""
    import numpy as np

    a = int(np.searchsorted(doc_ids, lo, side="right"))
    b = int(np.searchsorted(doc_ids, hi, side="right"))
    return doc_ids[a:b], (freqs[a:b] if freqs is not None else None)


def allgather_topn(scores, doc_ids, count: int, group=None):
    """This rank's top-N (scores f64 [n], docIds i64 [n], `count` valid) -> ([G,n], [G,n], [G]) on every rank."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    cnt = torch.tensor([count], dtype=torch.int64, device=scores.device)
    ls = [torch.empty_like(scores) for _ in range(world)]
    li = [torch.empty_like(doc_ids) for _ in range(world)]
    lc = [torch.empty_like(cnt) for _ in range(world)]
    dist.all_gather(ls, scores.contiguous(), group=group)
    dist.all_gather(li, doc_ids.contiguous(), group=group)
    dist.all_gather(lc, cnt, group=group)
    return torch.stack(ls), torch.stack(li), torch.cat(lc)


def merge_topn(gath_scores, gath_ids, counts, n: int):
    """[G,per] gathered per-shard lists -> global top-n (ids uint64, scores f64) with II_MergeShardTopN."""
    import numpy as np

    from . import postings

    sc = np.ascontiguousarray(gath_scores.cpu().numpy(), dtype=np.float64)
    ids = np.ascontiguousarray(gath_ids.cpu().numpy()).astype(np.uint64)
    cn = np.ascontiguousarray(counts.cpu().numpy()).astype(np.uint64)
    out_i = np.zeros(n, dtype=np.uint64)
    out_s = np.zeros(n, dtype=np.float64)
    got = postings.lib().II_MergeShardTopN(sc.ctypes.data, ids.ctypes.data, cn.ctypes.data, sc.shape[0], sc.shape[1], n,
                                           out_i.ctypes.data, out_s.ctypes.data)
    return out_i[:got], out_s[:got]
