"""Torch restatement of the reference's training criterion: test infrastructure, like the stage references beside it.

Functional, no modules, no state; every function runs in the dtype of its inputs, so the GPU tests evaluate it in
float64 and differentiate it with torch autograd.  `file:line` refers to the reference checkout.

What pins it:
  * `charbonnier`, `criterion_rgb`, `temporal_rgb`, `flow_l1` restate utils.img2charbonier and the four helpers of
    ibrnet/criterion.py, which can be executed: tests/golden/loss_terms.pt holds their outputs on seeded inputs
    (tests/golden/make_golden_loss.py).
  * `distortion` restates torch_efficient_distloss.eff_distloss_native, a package that is not available here; it is
    checked against the O(S^2) definition (`distortion_pairwise`) instead.
  * The rest of `mono_step_loss` restates the inline block train.py:300-456, which is not a callable: it is pinned by
    reading only.
"""

import torch

TERM_NAMES = ("loss", "flow_loss", "disp_loss", "rgb_loss", "distortion_loss", "entropy_loss", "static_loss",
              "cycle_loss", "reg_loss")


def charbonnier(x, y, mask):
  """utils.py:32-39 with eps = 0.001 (ibrnet/criterion.py:19); mask [R]."""
  mask = mask.to(x.dtype)
  return (torch.sqrt((x - y) ** 2 + 0.001 ** 2) * mask[:, None]).sum() / (mask.sum() * x.shape[-1] + 1e-6)


def criterion_rgb(outputs, ray_batch, motion_mask=None):
  """Criterion.forward, ibrnet/criterion.py:25-38."""
  mask = outputs["mask"].to(outputs["rgb"].dtype)
  if motion_mask is not None:
    mask = mask * motion_mask.to(mask.dtype)
  return charbonnier(outputs["rgb"], ray_batch["rgb"].to(mask.dtype), mask)


def rgb_loss(pred_rgb, ray_batch, pred_mask):
  """compute_rgb_loss, ibrnet/criterion.py:58-62."""
  return charbonnier(pred_rgb, ray_batch["rgb"].to(pred_rgb.dtype), pred_mask)


def temporal_rgb(outputs, ray_batch, motion_mask=None):
  """compute_temporal_rgb_loss, ibrnet/criterion.py:42-56."""
  pred = outputs["rgb"]
  w = outputs["mask"].to(pred.dtype)
  if motion_mask is not None:
    w = w * motion_mask.to(pred.dtype)
  w = (w * outputs["occ_weight_map"].to(pred.dtype))[:, None].expand(-1, 3)
  return (w * torch.sqrt((pred - ray_batch["rgb"].to(pred.dtype)) ** 2 + 0.001 ** 2)).sum() / (w.sum() + 1e-8)


def flow_l1(render_flow, gt_flow, gt_mask):
  """compute_flow_loss, ibrnet/criterion.py:83-85; gt_mask [n,R,1]."""
  m = gt_mask.to(render_flow.dtype).expand(-1, -1, 2)
  return ((render_flow - gt_flow.to(render_flow.dtype)).abs() * m).sum() / (m.sum() + 1e-8)


def distortion(w, m, interval):
  """eff_distloss_native(w, m, interval) as train.py:421 uses it, in the cumulative-sum form: per ray
  2 sum_{i>=1} (w_i m_i W_{i-1} - w_i WM_{i-1}) + 1/3 sum_i interval_i w_i^2, W / WM the inclusive prefix sums of w /
  w m; mean over the rays."""
  wm = w * m
  W, WM = torch.cumsum(w, -1), torch.cumsum(wm, -1)
  inter = 2.0 * (wm[..., 1:] * W[..., :-1] - w[..., 1:] * WM[..., :-1]).sum(-1)
  intra = (interval * w ** 2).sum(-1) / 3.0
  return (inter + intra).mean()


def distortion_pairwise(w, m, interval):
  """The definition (mip-NeRF 360, eq. 15): sum_ij w_i w_j |m_i - m_j| + 1/3 sum_i w_i^2 interval_i, mean over rays."""
  pair = (w[..., :, None] * w[..., None, :] * (m[..., :, None] - m[..., None, :]).abs()).sum((-1, -2))
  return (pair + (interval * w ** 2).sum(-1) / 3.0).mean()


def step_weights(args, epoch):
  """train.py:302, :318, :331, :345, :354-357."""
  divisor = epoch // args.init_decay_epoch
  if args.anneal_cycle:
    w_cycle = min(0.5, args.w_cycle + divisor * args.cycle_factor)
  else:
    w_cycle = args.w_cycle
  return dict(divisor=divisor, dy_rgb=1.0 / 10.0 ** divisor, w_disp=args.w_disp / args.decay_rate ** divisor,
              w_flow=args.w_flow / args.decay_rate ** divisor, w_cycle=w_cycle,
              dynamic_rgb=epoch < args.init_decay_epoch, static_dy=divisor > 4)


def static_bootstrap_loss(ret, ray_batch):
  """train.py:187-196."""
  pred = ret["outputs_coarse_st"]["rgb"]
  mask = (1.0 - ray_batch["static_mask"].to(pred.dtype)) * ret["outputs_coarse_ref"]["mask"].to(pred.dtype)
  return rgb_loss(pred, ray_batch, mask)


def step_denominators(ret, ray_batch, args, epoch):
  """The quantities through which mono_step_loss couples rays: the normalisers of its terms and the counts of its
  means.  Each is built from supervision, from masks or from forward values the loss detaches (occ_weight_map,
  occ_weights, `ratio` in the static mask), so a ray-chunked evaluation computes them once over all rays and holds
  them fixed (tests/train_step_ref.py).  The rgb and disparity normalisers are left live: with the reference's
  detaches they carry no gradient, and a caller that removes one sees its effect."""
  ref, ref_dy = ret["outputs_coarse_ref"], ret["outputs_coarse_ref_dy"]
  anc, anc_dy = ret["outputs_coarse_anchor"], ret["outputs_coarse_anchor_dy"]
  dt = ref["rgb"].dtype
  sw = step_weights(args, epoch)
  motion = ray_batch["motion_mask"].to(dt)
  pred_mask = ref["mask"].to(dt)
  R = pred_mask.shape[0]
  sum_dy, sum_st = ref["weights_dy"].sum(-1), ref["weights_st"].sum(-1)
  ratio = (sum_dy / torch.clamp(sum_dy + sum_st, min=1e-9)).detach()
  smask = (1.0 - ray_batch["static_mask"].to(dt)) * pred_mask * (1.0 - ratio)
  sf = anc["sf_seq"]
  n, _, S, c = sf.shape
  flow_m = (pred_mask[None, :, None] * ray_batch["masks"].to(dt)).expand(-1, -1, 2)
  t_anc = anc["pts_traj_anchor"]
  d = dict(
      rgb_ref=pred_mask.sum() * 3 + 1e-6,  # charbonnier: mask.sum() * channels + 1e-6
      rgb_anchor=(anc["mask"].to(dt) * anc["occ_weight_map"].to(dt)).sum() * 3 + 1e-8,
      rgb_ref_dy=(ref_dy["mask"].to(dt) * motion).sum() * 3 + 1e-6,
      rgb_anchor_dy=(anc_dy["mask"].to(dt) * motion * anc_dy["occ_weight_map"].to(dt)).sum() * 3 + 1e-8,
      disp=pred_mask.sum() + 1e-8,
      flow=flow_m.sum() + 1e-8,
      cycle=anc["occ_weights"].to(dt).sum() * t_anc.shape[0] * t_anc.shape[-1] + 1e-8,
      n_rays=float(R), n_sf=float(n * R * S * c), n_sf_time=float((n - 1) * R * S * c),
      n_sf_space=float(n * R * (S - 1) * c),
      static=smask.sum() * 3 + 1e-6)
  if sw["dynamic_rgb"]:
    d["rgb_dynamic"] = (pred_mask * motion).sum() * 3 + 1e-6
  if sw["static_dy"]:
    d["static_dy"] = (smask * (ratio < 0.1).to(dt) + 1e-8).sum()
  return d


def mono_step_loss(ret, ray_batch, args, epoch, den=None):
  """train.py:300-456 -> (loss, dict of the scalars :458-464 logs plus cycle_loss and reg_loss).

  den: None, or step_denominators() of the whole batch when `ret` / `ray_batch` hold a chunk of its rays; the
  chunks' losses then sum to the batch's loss and their gradients to its gradient."""
  ref, ref_dy = ret["outputs_coarse_ref"], ret["outputs_coarse_ref_dy"]
  anc, anc_dy = ret["outputs_coarse_anchor"], ret["outputs_coarse_anchor_dy"]
  dt = ref["rgb"].dtype
  sw = step_weights(args, epoch)
  if den is None:
    den = step_denominators(ret, ray_batch, args, epoch)
  motion = ray_batch["motion_mask"].to(dt)
  pred_mask = ref["mask"].to(dt)
  gt = ray_batch["rgb"].to(dt)
  charb = lambda x: torch.sqrt((x - gt) ** 2 + 0.001 ** 2)
  # rgb, :304-328 (criterion_rgb, temporal_rgb, rgb_loss with the normalisers of `den`)
  rgb = (charb(ref["rgb"]) * pred_mask[:, None]).sum() / den["rgb_ref"]
  w_anc = anc["mask"].to(dt) * anc["occ_weight_map"].to(dt)
  rgb = rgb + (charb(anc["rgb"]) * w_anc[:, None]).sum() / den["rgb_anchor"]
  if sw["dynamic_rgb"]:
    rgb = rgb + (charb(ref["rgb_dy"]) * (pred_mask * motion)[:, None]).sum() / den["rgb_dynamic"]
  rgb = rgb + (charb(ref_dy["rgb"]) * (ref_dy["mask"].to(dt) * motion)[:, None]).sum() / den["rgb_ref_dy"] * sw["dy_rgb"]
  w_anc_dy = anc_dy["mask"].to(dt) * motion * anc_dy["occ_weight_map"].to(dt)
  rgb = rgb + (charb(anc_dy["rgb"]) * w_anc_dy[:, None]).sum() / den["rgb_anchor_dy"] * sw["dy_rgb"]
  # disparity, :331-342
  pred_disp = 1.0 / torch.clamp(ref["depth"], min=1e-2)
  disp = sw["w_disp"] * ((pred_disp - ray_batch["disp"].to(dt)).abs() * pred_mask).sum() / den["disp"]
  # flow, :345-351
  m = (pred_mask[None, :, None] * ray_batch["masks"].to(dt)).expand(-1, -1, 2)
  flow = sw["w_flow"] * ((ref["render_flows"] - ray_batch["flows"].to(dt)).abs() * m).sum() / den["flow"]
  # trajectory cycle, :359-371
  t_ref, t_anc = anc["pts_traj_ref"], anc["pts_traj_anchor"]
  occ = anc["occ_weights"].to(dt)[None, ..., None].expand(t_anc.shape[0], -1, -1, t_anc.shape[-1])
  cycle = sw["w_cycle"] * ((t_ref - t_anc).abs() * occ).sum() / den["cycle"]
  # scene-flow regularisers, :374-397
  sf = anc["sf_seq"]
  reg = args.w_reg * sf.abs().sum() / den["n_sf"]
  reg = reg + args.w_reg * 0.5 * ((sf[:-1] - sf[1:]) ** 2).sum() / den["n_sf_time"]
  reg = reg + args.w_reg * (sf[:, :, 1:] - sf[:, :, :-1]).abs().sum() / den["n_sf_space"]
  # weight entropy, :400-413
  sum_dy, sum_st = ref["weights_dy"].sum(-1), ref["weights_st"].sum(-1)
  ratio = sum_dy / torch.clamp(sum_dy + sum_st, min=1e-9)
  ent = -(ratio * torch.log(ratio + 1e-9) + (1.0 - ratio) * torch.log(1.0 - ratio + 1e-9))
  ent = args.w_skew_entropy * ent.sum() / den["n_rays"]
  # distortion, :416-423
  s = ref["s_vals"].to(dt)
  dist = args.w_distortion * distortion(ref["weights"][:, :-1], (s[:, 1:] + s[:, :-1]) * 0.5,
                                        s[:, 1:] - s[:, :-1]) * (s.shape[0] / den["n_rays"])
  # adaptive static loss, :426-445
  smask = (1.0 - ray_batch["static_mask"].to(dt)) * pred_mask * (1.0 - ratio).detach()
  static = (charb(ref["rgb_static"]) * smask[:, None]).sum() / den["static"]
  if sw["static_dy"]:
    m2 = (smask * (ratio < 0.1).to(dt)).detach()
    static = static + 0.1 * (sum_dy * m2).abs().sum() / den["static_dy"]
  loss = rgb + cycle + flow + disp + reg + ent + dist + static  # :447-456
  vals = (loss, flow, disp, rgb, dist, ent, static, cycle, reg)
  return loss, {k: v.detach() for k, v in zip(TERM_NAMES, vals)}
