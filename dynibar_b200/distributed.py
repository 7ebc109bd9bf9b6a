"""Multi-GPU ray sharding (SURVEY.md 8(e)).

Rays are independent: a frame's pixel list is block-partitioned across the
ranks of one node (one process per GPU), every rank renders its block with zero
communication, and ONE gather of the rendered pixels (rgb, depth, mask: 5
floats per ray) brings the frame to rank 0 over NVLink/NVSwitch (NCCL) -- the
replacement for the reference's per-module-call `nn.DataParallel`
scatter/gather (ibrnet/model.py:130-159).  Source images / feature maps /
weights are replicated per rank (each rank can run the 2-D encoder itself, or
rank 0 broadcasts them once per frame with `broadcast_frame_inputs`).

Backend-agnostic (`nccl` on GPUs; the host logic is tested with `gloo`).
"""

import torch
import torch.distributed as dist

_RAY_KEYS_1 = ("ray_o", "ray_d", "uv_grid", "rgb", "disp", "motion_mask", "static_mask", "camera_index")


def shard_bounds(n_rays, rank, world):
  """Contiguous block [lo, hi) of rank `rank`; blocks differ by at most one ray."""
  base, rem = divmod(n_rays, world)
  lo = rank * base + min(rank, rem)
  return lo, lo + base + (1 if rank < rem else 0)


def shard_ray_batch(ray_batch, rank, world):
  """This rank's slice of a full-frame ray batch (per-ray tensors are sliced,
  per-frame tensors are shared)."""
  n = ray_batch["ray_o"].shape[0]
  lo, hi = shard_bounds(n, rank, world)
  out = dict(ray_batch)
  for k, v in ray_batch.items():
    if not torch.is_tensor(v):
      continue
    if k in _RAY_KEYS_1 and v.shape[0] == n:
      out[k] = v[lo:hi].contiguous()
    elif k in ("flows", "masks") and v.dim() == 3 and v.shape[1] == n:
      out[k] = v[:, lo:hi].contiguous()
  return out, (lo, hi)


def gather_pixels(pixels, n_rays, dst=0, group=None):
  """pixels [n_local, C] of every rank -> [n_rays, C] on `dst` (None elsewhere).
  Shards may differ by one ray, so blocks are padded to the largest shard."""
  world = dist.get_world_size(group)
  rank = dist.get_rank(group)
  if world == 1:
    return pixels
  per = (n_rays + world - 1) // world
  C = pixels.shape[1]
  buf = torch.zeros(per, C, dtype=pixels.dtype, device=pixels.device)
  buf[:pixels.shape[0]] = pixels
  out = [torch.empty_like(buf) for _ in range(world)] if rank == dst else None
  dist.gather(buf, out, dst=dst, group=group)
  if rank != dst:
    return None
  parts = []
  for r in range(world):
    lo, hi = shard_bounds(n_rays, r, world)
    parts.append(out[r][:hi - lo])
  return torch.cat(parts, 0)


def broadcast_frame_inputs(tensors, src=0, group=None):
  """Once per frame: source images / feature maps / cameras from the rank that
  produced them (in place)."""
  if dist.get_world_size(group) == 1:
    return tensors
  for t in tensors:
    if t is not None:
      dist.broadcast(t, src=src, group=group)
  return tensors


def render_frame_sharded(render_fn, ray_batch, group=None, dst=0):
  """render_fn(local_ray_batch) -> [n_local, C] pixel tensor.  Returns the
  assembled [n_rays, C] frame on `dst`, None on the other ranks."""
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  rank = dist.get_rank(group) if dist.is_initialized() else 0
  n = ray_batch["ray_o"].shape[0]
  local, _ = shard_ray_batch(ray_batch, rank, world)
  px = render_fn(local)
  if world == 1:
    return px
  return gather_pixels(px, n, dst=dst, group=group)


def allreduce_gradients(params, group=None, average=True):
  """Training (SURVEY 8(e), BASELINE config 3): every rank renders its share of the N_rand rays and the gradients
  of the ~1.6 M parameters are summed (averaged) with ONE all-reduce per step over a flat bucket -- the reference
  never all-reduces (train.py:769-774 creates a process group but wraps nothing in DDP).  `params`: iterable of
  tensors whose .grad to reduce in place (parameters that received no gradient on this rank contribute zeros).
  Returns the number of elements reduced."""
  params = [p for p in params if p.requires_grad]
  if not params:
    return 0
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  for p in params:
    if p.grad is None:
      p.grad = torch.zeros_like(p)
  if world == 1:
    return sum(p.numel() for p in params)
  flat = torch.cat([p.grad.reshape(-1) for p in params])
  dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
  if average:
    flat /= world
  o = 0
  for p in params:
    n = p.numel()
    p.grad.copy_(flat[o:o + n].view_as(p.grad))
    o += n
  return o
