"""Multi-GPU data path: images are sharded over ranks (one process per GPU, weights replicated); the ONLY collective is a
fixed-shape all-gather of the per-image detections over NCCL/NVLink (gloo in the CPU tests) — ONE collective per step.

It replaces the reference's pickled, variable-length ``all_gather`` of whole-dataset prediction dicts
(maskrcnn_benchmark/utils/comm.py:61-102, engine/inference.py:293-312): after the top-k cut every image has at most
``max_out`` rows of (x1, y1, x2, y2, score, label); the count of valid rows rides in an extra row of the same buffer
(``mqdet_gather_detections`` with ``det_rows = max_out + 1``), so the exchange is ONE ``[B_local, max_out + 1, 6]`` fp32
buffer per rank (24.8 KB at B_local = 8, max_out = 128) — latency-bound, never bandwidth-bound.
"""
import torch
import torch.distributed as dist


def shard_indices(num_images, rank, world):
    """image i -> rank i % world (DistributedSampler order, data/build.py:196-198)."""
    return list(range(rank, num_images, world))


def all_gather_detections(det, num, group=None):
    """det [B_local, max_out, 6], num [B_local] (device or CPU tensors) -> (det_all [world*B_local, max_out, 6],
    num_all [world*B_local]) in RANK-MAJOR order; identity when no process group is initialised."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return det, num
    det_all, num_all = unpack(all_gather_packed(pack(det, num), group))
    return det_all, num_all.to(num.dtype)


def pack(det, num):
    """det [B, max_out, 6] + num [B] -> packed [B, max_out + 1, 6] (row max_out = (count, 0, ...)); host/test helper — the
    device path gets the packed buffer straight from ``mqdet_gather_detections``."""
    packed = torch.zeros((det.shape[0], det.shape[1] + 1, 6), dtype=det.dtype, device=det.device)
    packed[:, :-1] = det
    packed[:, -1, 0] = num.to(det.dtype)
    return packed


def unpack(packed):
    """packed [B, max_out + 1, 6] -> (det view [B, max_out, 6], num int32 [B])."""
    return packed[:, :-1], packed[:, -1, 0].round().to(torch.int32)


def all_gather_packed(packed, group=None, out=None):
    """ONE collective: packed [B_local, max_out + 1, 6] -> [world * B_local, max_out + 1, 6] in RANK-MAJOR order; identity
    when no process group is initialised.  ``out`` = preallocated destination (CUDA-graph friendly)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return packed
    world = dist.get_world_size(group)
    if out is None:
        out = torch.empty((world * packed.shape[0],) + tuple(packed.shape[1:]), dtype=packed.dtype, device=packed.device)
    dist.all_gather_into_tensor(out, packed.contiguous(), group=group)
    return out


def unshard(det_all, num_all, num_images, world):
    """rank-major gathered rows -> original image order for images sharded with ``shard_indices``."""
    per = det_all.shape[0] // world
    order = []
    for r in range(world):
        order += [(i, r * per + k) for k, i in enumerate(shard_indices(num_images, r, world))]
    order.sort()
    idx = torch.tensor([j for _, j in order], dtype=torch.long, device=det_all.device)
    return det_all.index_select(0, idx), num_all.index_select(0, idx)


# ---- many-category prompts: the chunks of the vocabulary (text-token columns) shard over ranks --------------------------
def shard_chunks(num_chunks, rank, world):
    """prompt chunk c -> rank c % world (SURVEY.md §8e, second partition axis: the reference evaluates the 31 LVIS chunks
    one after the other on every rank, engine/inference.py:605-625)."""
    return list(range(rank, num_chunks, world))


def all_gather_chunks(packed_local, num_chunks, group=None):
    """packed_local [n_local, B, max_out + 1, 6] = the packed detections of this rank's chunks (``shard_chunks`` order) ->
    [num_chunks, B, max_out + 1, 6] in chunk order on every rank, with ONE fixed-shape all-gather (ranks with one chunk
    fewer send a zero block: count 0)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return packed_local
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    per = -(-num_chunks // world)
    buf = packed_local
    if packed_local.shape[0] < per:
        buf = torch.zeros((per,) + tuple(packed_local.shape[1:]), dtype=packed_local.dtype, device=packed_local.device)
        buf[: packed_local.shape[0]] = packed_local
    out = torch.empty((world * per,) + tuple(buf.shape[1:]), dtype=buf.dtype, device=buf.device)
    dist.all_gather_into_tensor(out, buf.contiguous(), group=group)
    idx = torch.tensor([(c % world) * per + c // world for c in range(num_chunks)], dtype=torch.long, device=out.device)
    return out.index_select(0, idx)


def all_reduce_loss_normalizers(buf, group=None):
    """The ATSS loss normalisers (number of positives, sum of centerness targets; loss.py:1149-1151, :1188) summed over the ranks
    in place with ONE collective, between the target assignment and the losses: ``buf`` = ``ops.atss_targets(...)["norm"][:2]``
    (a view: the rank-local copies in ``norm[2:]`` stay untouched).  Identity when no process group is initialised."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return buf
    dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
    return buf


def all_reduce_gradients(grads, group=None, average=True):
    """Data-parallel gradient exchange of the modulated pre-training (the reference wraps the model in DistributedDataParallel,
    tools/train_net.py:96-103; only the ~45.7 M GCP / PreSelect parameters carry gradients): ALL gradient tensors of a step are packed
    into ONE flat fp32 buffer and reduced by ONE collective (NCCL all-reduce over NVLink; 183 MB), then averaged over the ranks like
    DDP does and scattered back into the given tensors in place.  ``grads``: {name: fp32 tensor}; iteration order = key order, which
    must be the same on every rank (it is: ``QVBertModelTrain.backward`` builds the dict deterministically).  Identity when no
    process group is initialised."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return grads
    world = dist.get_world_size(group)
    keys = sorted(grads)
    flat = torch.cat([grads[k].reshape(-1).float() for k in keys])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    if average:
        flat.div_(world)
    off = 0
    for k in keys:
        n = grads[k].numel()
        grads[k].copy_(flat[off:off + n].view_as(grads[k]))
        off += n
    return grads
