"""The training criterion of a DynibarMono step on the GPU (row f2).

`mono_step_loss` is the loss block of the reference's train() (train.py:300-456) and `static_bootstrap_loss` the one of
its static warm-up (train.py:187-196), computed from the dicts `render_ray.render_rays_mono(is_train=True)` returns and
the batch `RaySamplerSingleImage.random_sample` returns.  The names train.py imports for its loss -- `Criterion`,
`compute_rgb_loss`, `compute_temporal_rgb_loss`, `compute_flow_loss` (ibrnet/criterion.py) and `eff_distloss_native`
(the torch_efficient_distloss package) -- are here as well.

All of them are the same pair of kernels (csrc/loss.cu: `dyn_mono_loss`, `dyn_mono_loss_backward`) with different
terms switched on: two launches forward, one backward, no float atomics (the same inputs give the same bits), nothing
read back to the host.  CUDA tensors only.
"""

import torch

from dynibar_b200 import _lib
from dynibar_b200 import autograd as ag

# term indices of dyn_mono_loss (include/dynibar_b200.h)
RGB_REF, RGB_ANCHOR, RGB_DYNAMIC, RGB_REF_DY, RGB_ANCHOR_DY, STATIC = range(6)
DISP, FLOW, CYCLE, REG_ABS, REG_TIME, REG_SPACE, ENTROPY, DISTORTION, STATIC_DY = range(6, 15)
# the scalars train.py:458-464 logs, then the two it does not, in the order of out[0:9]
TERM_NAMES = ("loss", "flow_loss", "disp_loss", "rgb_loss", "distortion_loss", "entropy_loss", "static_loss",
              "cycle_loss", "reg_loss")
COMPONENTS = 9  # out[COMPONENTS + k]: term k before its weight
_CHARBONNIER_EPS, _TEMPORAL_EPS = 1e-6, 1e-8  # utils.py:39 (TINY_NUMBER), criterion.py:55


def _weights(terms):
  """dyn_mono_loss_weights with the given {term: weight} present."""
  wt = _lib.MonoLossWeights()
  for k, w in terms.items():
    wt.terms |= 1 << k
    wt.w[k] = w
  for k in range(_lib.LOSS_RGB_SLOTS):
    wt.rgb_eps[k] = _TEMPORAL_EPS if k in (RGB_ANCHOR, RGB_ANCHOR_DY) else _CHARBONNIER_EPS
  return wt


def step_weights(args, epoch):
  """The weight and the presence of every term at `epoch` (train.py:302-357, :374, :413, :420, :437), as the struct the
  kernels take by value."""
  divisor = epoch // args.init_decay_epoch
  dy_decay = 1.0 / 10.0 ** divisor                   # dynamic_rgb_decay_rate, :318-328
  data_decay = 1.0 / args.decay_rate ** divisor      # :331, :345
  w_cycle = min(0.5, args.w_cycle + divisor * args.cycle_factor) if args.anneal_cycle else args.w_cycle
  terms = {RGB_REF: 1.0, RGB_ANCHOR: 1.0, RGB_REF_DY: dy_decay, RGB_ANCHOR_DY: dy_decay, STATIC: 1.0,
           DISP: args.w_disp * data_decay, FLOW: args.w_flow * data_decay, CYCLE: w_cycle,
           REG_ABS: args.w_reg, REG_TIME: 0.5 * args.w_reg, REG_SPACE: args.w_reg,
           ENTROPY: args.w_skew_entropy, DISTORTION: args.w_distortion}
  if epoch < args.init_decay_epoch:
    terms[RGB_DYNAMIC] = 1.0
  if divisor > 4:
    terms[STATIC_DY] = 0.1
  return _weights(terms)


def _slot(*factors, flags=0):
  """Per-ray weight of an rgb term: the product of a bool mask and up to two float factors (None = absent)."""
  slot, floats = {"flags": flags}, []
  for f in factors:
    if f is None:
      continue
    if f.dtype == torch.bool and "mask" not in slot:
      slot["mask"] = f.reshape(-1)
    else:
      floats.append(f.reshape(-1))
  if len(floats) > 2:
    raise ValueError("criterion: at most two float factors per rgb term")
  slot.update(zip(("w0", "w1"), floats))
  return slot


def mono_step_loss(ret, ray_batch, args, epoch):
  """The loss of one training step (train.py:300-456) -> (loss, terms).

  ret: what render_rays_mono(is_train=True) returned; ray_batch: what RaySamplerSingleImage.random_sample returned
  (rgb, disp, motion_mask, static_mask, flows, masks); args: w_disp, w_flow, w_cycle, cycle_factor, anneal_cycle, w_reg,
  w_skew_entropy, w_distortion, decay_rate, init_decay_epoch.  loss: 0-d device tensor to call backward() on; terms:
  detached 0-d device tensors under the keys of TERM_NAMES.  Nothing is read back to the host."""
  out = mono_step_table(ret, ray_batch, args, epoch)
  return out[0], dict(zip(TERM_NAMES, out.detach()[:len(TERM_NAMES)].unbind()))


def mono_step_table(ret, ray_batch, args, epoch):
  """Everything the forward kernels write for a step, one [40] device tensor: [0:9] the scalars of TERM_NAMES (element 0,
  the loss, is the differentiable one), [COMPONENTS + k] term k before its weight (k: the indices above)."""
  wt, fixed, inputs = _step_call(ret, ray_batch, args, epoch)
  return ag.mono_loss(wt, fixed, **inputs)


def _step_call(ret, ray_batch, args, epoch):
  """(weights, fixed, differentiable inputs) of the criterion call of a step (train.py:300-456)."""
  ref, ref_dy = ret["outputs_coarse_ref"], ret["outputs_coarse_ref_dy"]
  anc, anc_dy = ret["outputs_coarse_anchor"], ret["outputs_coarse_anchor_dy"]
  wt = step_weights(args, epoch)
  if anc["pts_traj_ref"].shape[0] == 0:  # no anchor offset within +-3 frames: the term is 0
    wt.terms &= ~(1 << CYCLE)
  R, S = ref["weights"].shape
  motion = ray_batch["motion_mask"].float()
  fixed = {
      "R": R, "S": S, "gt_rgb": ray_batch["rgb"],
      "slot%d" % RGB_REF: _slot(ref["mask"]),
      "slot%d" % RGB_ANCHOR: _slot(anc["mask"], anc["occ_weight_map"]),
      "slot%d" % RGB_DYNAMIC: _slot(ref["mask"], motion),
      "slot%d" % RGB_REF_DY: _slot(ref_dy["mask"], motion),
      "slot%d" % RGB_ANCHOR_DY: _slot(anc_dy["mask"], motion, anc_dy["occ_weight_map"]),
      # (1 - static_mask) * mask * (1 - weights_ratio).detach(), :426-428
      "slot%d" % STATIC: _slot(ref["mask"], ray_batch["static_mask"].float(),
                               flags=_lib.LOSS_SLOT_COMPLEMENT_W0 | _lib.LOSS_SLOT_TIMES_ONE_MINUS_RATIO),
      "gt_disp": ray_batch["disp"], "ray_mask": ref["mask"],
      "gt_flows": ray_batch["flows"], "flow_masks": ray_batch["masks"],
      "occ_weights": anc["occ_weights"], "s_vals": ref["s_vals"], "dist_n": S - 1,
  }
  return wt, fixed, dict(
      rgb0=ref["rgb"], rgb1=anc["rgb"], rgb2=ref["rgb_dy"] if (wt.terms >> RGB_DYNAMIC) & 1 else None,
      rgb3=ref_dy["rgb"], rgb4=anc_dy["rgb"], rgb5=ref["rgb_static"], depth=ref["depth"], flows=ref["render_flows"],
      weights=ref["weights"], weights_dy=ref["weights_dy"], weights_st=ref["weights_st"],
      traj_ref=anc["pts_traj_ref"], traj_anchor=anc["pts_traj_anchor"], sf_seq=anc["sf_seq"])


def static_bootstrap_loss(ret, ray_batch):
  """The loss of the static warm-up (train.py:187-196): Charbonnier of outputs_coarse_st['rgb'] under
  (1 - static_mask) * outputs_coarse_ref['mask']."""
  wt, fixed, inputs = _bootstrap_call(ret, ray_batch)
  return ag.mono_loss(wt, fixed, **inputs)[0]


def _bootstrap_call(ret, ray_batch):
  pred = ret["outputs_coarse_st"]["rgb"]
  slot = _slot(ret["outputs_coarse_ref"]["mask"], ray_batch["static_mask"].float(),
               flags=_lib.LOSS_SLOT_COMPLEMENT_W0)
  return _rgb_call(STATIC, pred, ray_batch["rgb"], slot)


# ---- the criterion of a batch evaluated in ray slices (dynibar_b200/train_step.py) ----------------------------------
# The terms couple rays only through denominators built from supervision, masks and detached forward values, so a
# batch's loss and gradient come from: rows of every slice (pass 1, no gradient) -> one finish with the batch's
# dimensions -> each slice's backward against that table.  `bootstrap` selects static_bootstrap_loss's single term
# instead of mono_step_loss's.
def _call(ret, ray_batch, args, epoch, bootstrap):
  return _bootstrap_call(ret, ray_batch) if bootstrap else _step_call(ret, ray_batch, args, epoch)


def slice_rows(ret, ray_batch, args, epoch, partial, first_ray, bootstrap=False):
  """Writes the criterion rows of one ray slice (`ret` its render output, `ray_batch` its rays and supervision) that
  starts at ray `first_ray` of the batch into `partial` (uint8, dyn_mono_loss_workspace_bytes(R_batch) bytes).
  -> (weights, (S, K, n_sf)) for batch_table."""
  wt, fixed, inputs = _call(ret, ray_batch, args, epoch, bootstrap)
  return wt, ag.mono_loss_rows(wt, fixed, partial, first_ray, **inputs)


def batch_table(partial, weights, R, dims):
  """The [40] table of mono_step_table (or the bootstrap's) for the R-ray batch whose rows `partial` holds."""
  return ag.mono_loss_finish(partial, weights, R, *dims)


def slice_loss(ret, ray_batch, args, epoch, table, bootstrap=False):
  """0-d tensor whose backward adds one ray slice's share of d(batch loss) / d(render outputs); its value is the
  batch's loss.  `table`: batch_table of the batch."""
  wt, fixed, inputs = _call(ret, ray_batch, args, epoch, bootstrap)
  return ag.mono_loss(wt, dict(fixed, table=table), **inputs)[0]


def _rgb_call(k, pred, gt, slot):
  return _weights({k: 1.0}), {"R": pred.shape[0], "S": 2, "gt_rgb": gt, "slot%d" % k: slot}, {"rgb%d" % k: pred}


def _rgb_term(k, pred, gt, slot):
  wt, fixed, inputs = _rgb_call(k, pred, gt, slot)
  return ag.mono_loss(wt, fixed, **inputs)[0]


class Criterion(torch.nn.Module):
  """ibrnet/criterion.py:21-38: Charbonnier of outputs['rgb'] under outputs['mask'] (* motion_mask)."""

  def forward(self, outputs, ray_batch, motion_mask=None):
    return _rgb_term(RGB_REF, outputs["rgb"], ray_batch["rgb"], _slot(outputs["mask"], motion_mask))


def compute_rgb_loss(pred_rgb, ray_batch, pred_mask):
  """ibrnet/criterion.py:58-62."""
  return _rgb_term(RGB_REF, pred_rgb, ray_batch["rgb"], _slot(pred_mask))


def compute_temporal_rgb_loss(outputs, ray_batch, motion_mask=None):
  """ibrnet/criterion.py:42-56: weighted by mask (* motion_mask) * occ_weight_map."""
  return _rgb_term(RGB_ANCHOR, outputs["rgb"], ray_batch["rgb"],
                   _slot(outputs["mask"], motion_mask, outputs["occ_weight_map"]))


def compute_flow_loss(render_flow, gt_flow, gt_mask):
  """ibrnet/criterion.py:83-85: render_flow, gt_flow [n,R,2], gt_mask [n,R,1]."""
  fixed = {"R": render_flow.shape[1], "S": 2, "gt_flows": gt_flow, "flow_masks": gt_mask}
  return ag.mono_loss(_weights({FLOW: 1.0}), fixed, flows=render_flow)[0]


def eff_distloss_native(w, m, interval):
  """The distortion loss of mip-NeRF 360 as train.py:421 calls it (torch_efficient_distloss.eff_distloss_native):
  w, m, interval [R,N] -> mean over the rays of sum_ij w_i w_j |m_i - m_j| + 1/3 sum_i w_i^2 interval_i; the gradient
  goes to w."""
  w = w.contiguous()
  fixed = {"R": w.shape[0], "S": 2, "dist_n": w.shape[1], "dist_m": m, "dist_interval": interval}
  return ag.mono_loss(_weights({DISTORTION: 1.0}), fixed, weights=w)[0]
