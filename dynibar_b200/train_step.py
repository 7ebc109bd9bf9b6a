"""One monocular training step's forward and backward in ray slices, so that the shipped batch (N_rand 3072 x 64
samples, 14 static views) trains on one 80 GB GPU.

`mono_step_backward` replaces train.py's render_rays_mono(is_train=True) / loss / loss.backward() (and the static
warm-up's, train.py:169-198).  The criterion couples rays only through normalisers and counts built from supervision,
masks and forward values the reference detaches (occ_weight_map, 1 - weights_ratio, the m2 mask of the late static
term), so the whole batch's gradient is:
  pass 1  for each slice, the training forward under no_grad and its criterion rows (criterion.slice_rows); then one
          finish over the batch's rows (criterion.batch_table): the batch's loss, terms and denominators;
  pass 2  for each slice, the training forward with gradients, the slice's loss backward against the batch table
          (criterion.slice_loss) and the network backward; the slice's graph is freed before the next one.
The feature maps enter as detached leaves; their gradients add up over the slices and reach the encoder in one
backward at the end.  Peak memory is the encoder's activations, one slice's graph and the batch.
"""

import torch

from dynibar_b200 import _lib, criterion
from dynibar_b200 import render_ray as rr

# row counts at which the library's training products change implementation (tests/train_stage_ref.dispatch):
# forward products go to the tensor cores from 128 rows, backward products from 2048
FORWARD_ROWS, BACKWARD_ROWS = 128, 2048
# per-ray inputs of a ray batch: [R, ...] and [n, R, ...]
_RAY_KEYS = ("ray_o", "ray_d", "uv_grid", "rgb", "disp", "motion_mask", "static_mask")
_RAY_KEYS_AXIS1 = ("flows", "masks")


def _sides(rays, S):
  """Which side of every row-count threshold a slice of `rays` rays falls on: per-ray rows (R) and per-point rows
  (R S) against the forward and the backward threshold."""
  return tuple(rows >= lim for lim in (FORWARD_ROWS, BACKWARD_ROWS) for rows in (rays, rays * S))


def slice_plan(R, slice_rays, S):
  """[(lo, hi)] ray spans of a batch of R rays with S samples in slices of at most `slice_rays` rays.

  One span when R <= slice_rays.  Otherwise n near-equal slices, every boundary on a multiple of 8 rays (a slice's
  criterion rows are then the batch's rows), n the least count for which every slice falls on the same side as the
  batch of each row-count threshold, so that a slice runs the products the whole batch would run.  One exception:
  a batch of BACKWARD_ROWS rays or more in slices below it runs its per-ray backward products (the products over R
  rows: ref_feature_fc, rgb_fc.0's direction columns) in fp32 instead of on the tensor cores; all its slices do the
  same.  Such a batch does not fit one slice's memory anyway at the shipped sizes.
  Raises ValueError when no plan exists."""
  R, slice_rays, S = int(R), int(slice_rays), int(S)
  if R <= 0 or slice_rays <= 0 or S <= 0:
    raise ValueError("slice_plan: R, slice_rays and S must be positive, got %d, %d, %d" % (R, slice_rays, S))
  if R <= slice_rays:
    return [(0, R)]
  want = _sides(R, S)
  for n in range(-(-R // slice_rays), R // 8 + 1):
    size = -(-R // (8 * n)) * 8
    spans = [(lo, min(R, lo + size)) for lo in range(0, R, size)]
    if size > slice_rays or len(spans) != n:
      continue
    sides = {_sides(hi - lo, S) for lo, hi in spans}
    # the per-ray backward threshold (index 2) only has to agree across the slices
    if len(sides) == 1 and all(a == b for i, (a, b) in enumerate(zip(next(iter(sides)), want)) if i != 2):
      return spans
  raise ValueError("slice_plan: no plan of slices of at most %d rays for %d rays x %d samples keeps every slice on "
                   "the batch's side of the row-count thresholds %d / %d" % (slice_rays, R, S, FORWARD_ROWS,
                                                                              BACKWARD_ROWS))


def _slice_batch(ray_batch, lo, hi):
  rb = dict(ray_batch)
  for k in _RAY_KEYS:
    if rb.get(k) is not None:
      rb[k] = ray_batch[k][lo:hi]
  for k in _RAY_KEYS_AXIS1:
    if rb.get(k) is not None:
      rb[k] = ray_batch[k][:, lo:hi]
  return rb


def mono_step_backward(frame_idx, time_embedding, time_offset, ray_batch, model, featmaps, projector, N_samples, args,
                       epoch, *, slice_rays=1024, bootstrap=False, inv_uniform=True, det=False, num_vv=2, jitter=None,
                       precision=None):
  """Forward and backward of one training step (train.py:283-466; with bootstrap=True the static warm-up, :169-198:
  is_train=False, static loss only) -> (loss, terms), detached device tensors; nothing is read back to the host.

  Adds the step's gradient into .grad of every tensor that requires grad (the parameters of the model's nets,
  trajectory_basis, and through `featmaps` the encoder); zeroes nothing and steps no optimizer.  The arguments are
  render_rays_mono's and mono_step_loss's.  The batch runs in slices of at most `slice_rays` rays (slice_plan); a batch
  that fits one slice runs exactly render_rays_mono, the loss and backward.  With det=False and no `jitter` the
  samples' jitter is drawn once for the batch, so the result does not depend on the slicing.  terms: the keys of
  criterion.TERM_NAMES (bootstrap: "loss" and "static_loss")."""
  R = ray_batch["ray_o"].shape[0]
  spans = slice_plan(R, slice_rays, N_samples)
  is_train = not bootstrap
  if len(spans) == 1:
    ret = rr.render_rays_mono(frame_idx, time_embedding, time_offset, ray_batch, model, featmaps, projector, N_samples,
                              args, inv_uniform=inv_uniform, det=det, is_train=is_train, num_vv=num_vv, jitter=jitter,
                              precision=precision)
    if bootstrap:
      loss = criterion.static_bootstrap_loss(ret, ray_batch)
      terms = {"loss": loss.detach(), "static_loss": loss.detach()}
    else:
      loss, terms = criterion.mono_step_loss(ret, ray_batch, args, epoch)
    del ret
    loss.backward()
    return loss.detach(), terms

  if not det and jitter is None:
    jitter = torch.rand(R, N_samples, device=ray_batch["ray_o"].device)
  leaves = tuple(None if f is None else f.detach().requires_grad_(f.requires_grad) for f in featmaps)

  def render(lo, hi):
    return rr._render_mono_train(frame_idx, time_embedding, time_offset, _slice_batch(ray_batch, lo, hi), model,
                                 leaves, N_samples, args, inv_uniform, det, is_train, num_vv,
                                 None if jitter is None else jitter[lo:hi])

  with rr.precision_scope(precision):
    table = batch_table(render, ray_batch, spans, args, epoch, bootstrap)
    for lo, hi in spans:  # pass 2: each slice's forward and backward against the batch table
      loss = criterion.slice_loss(render(lo, hi), _slice_batch(ray_batch, lo, hi), args, epoch, table, bootstrap)
      loss.backward()
      del loss
  grads = [(f, l.grad) for f, l in zip(featmaps, leaves) if l is not None and l.grad is not None]
  if grads:
    torch.autograd.backward([f for f, _ in grads], [g for _, g in grads])
  table = table.detach()
  if bootstrap:
    return table[0], {"loss": table[0], "static_loss": table[0]}
  return table[0], dict(zip(criterion.TERM_NAMES, table[:len(criterion.TERM_NAMES)].unbind()))


def batch_table(render, ray_batch, spans, args, epoch, bootstrap):
  """Pass 1: the training forward of every span under no_grad (`render(lo, hi)` -> its output dicts), its criterion
  rows, then the batch's [40] table (criterion.mono_step_table's layout)."""
  R = spans[-1][1]
  partial = torch.empty(int(_lib.lib.dyn_mono_loss_workspace_bytes(R)), dtype=torch.uint8,
                        device=ray_batch["ray_o"].device)
  with torch.no_grad():
    for lo, hi in spans:
      wt, dims = criterion.slice_rows(render(lo, hi), _slice_batch(ray_batch, lo, hi), args, epoch, partial, lo,
                                      bootstrap)
    return criterion.batch_table(partial, wt, R, dims)
