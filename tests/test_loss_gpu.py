"""dynibar_b200.criterion on the GPU against the torch restatement of the reference's criterion (tests/loss_ref.py)
evaluated in float64 on the same inputs, and differentiated by torch autograd.

The inputs are the output dicts of a real `render_rays_mono(is_train=True)` call on the training scene of
test_train_gpu.py (so masks, occ_weights and the number K of cycle offsets are what training sees), cut loose from the
renderer as leaves; supervision is seeded (scenes.sampler_data).  Bars: every component rel. 2e-5; gradients rtol 2e-4,
atol 1e-6 * max|g| per tensor.  The last test runs a whole training step.

The second half runs the criterion on generated inputs at the training batch (R = 3072, S = 64) and around the
kernels' chunk and block edges, with per-element ulp bars (see TOL there)."""

import copy
import math
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import loss_ref
import scenes
from dynibar_b200 import synthetic
from geometry_stage_ref import bar, excess

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
INIT_DECAY = 150

# what autograd reaches in train.py's own graph; everything else in the dicts must stay without a gradient
GRAD_KEYS = {
    "outputs_coarse_ref": ("rgb", "rgb_dy", "rgb_static", "depth", "render_flows", "weights", "weights_dy",
                           "weights_st"),
    "outputs_coarse_ref_dy": ("rgb",),
    "outputs_coarse_anchor": ("rgb", "pts_traj_ref", "pts_traj_anchor", "sf_seq"),
    "outputs_coarse_anchor_dy": ("rgb",),
}
NO_GRAD_KEYS = {"outputs_coarse_ref": ("s_vals",), "outputs_coarse_anchor": ("occ_weights", "occ_weight_map"),
                "outputs_coarse_anchor_dy": ("occ_weight_map",)}


def loss_args(args=None, **kw):
  a = dict(vars(args)) if args is not None else {}
  a.update(w_disp=5e-2, w_flow=5e-3, w_cycle=0.1, cycle_factor=0.1, anneal_cycle=True, w_reg=0.05,
           w_skew_entropy=1e-3, w_distortion=1e-3, decay_rate=10.0, init_decay_epoch=INIT_DECAY)
  a.update(kw)
  return SimpleNamespace(**a)


def supervision(batch, cfg, dev):
  """The keys RaySamplerSingleImage.random_sample adds for R seeded pixels of the frame's supervision."""
  data = scenes.sampler_data(batch, cfg["H"], cfg["W"], cfg["seed"])
  R = batch["ray_o"].shape[0]
  sel = torch.randperm(cfg["H"] * cfg["W"], generator=torch.Generator().manual_seed(cfg["seed"] + 7))[:R]
  flat = lambda t, c: t[0].reshape(-1, c)[sel]
  rb = {"rgb": flat(data["rgb"], 3), "disp": flat(data["disp"], 1)[:, 0],
        "motion_mask": flat(data["motion_mask"], 1)[:, 0], "static_mask": flat(data["static_mask"], 1)[:, 0],
        "flows": data["flows"][0].reshape(6, -1, 2)[:, sel], "masks": data["masks"][0].reshape(6, -1, 1)[:, sel]}
  return {k: v.to(dev) for k, v in rb.items()}


@pytest.fixture(scope="module")
def rendered():
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  cfg = dict(scenes.GOLDEN_CONFIGS["mono_train"])
  batch, feat_c, _, frame, t, offs, model, args = scenes.build(cfg)
  with torch.no_grad():
    model.motion_mlp.coeff_linear.weight.normal_(0.0, 0.05)
  dev = torch.device(DEV)
  m_dev = synthetic.model_to(model, dev)
  with torch.no_grad():
    ret = rr.render_rays_mono(frame, t, offs, synthetic.to_device(batch, dev), m_dev, synthetic.to_device(feat_c, dev),
                              Projector(dev), cfg["N_samples"], args, inv_uniform=True, det=True, is_train=True,
                              num_vv=cfg["num_vv"], precision="fp32")
  keep = ("outputs_coarse_ref", "outputs_coarse_ref_dy", "outputs_coarse_st", "outputs_coarse_anchor",
          "outputs_coarse_anchor_dy")
  ret = {o: {k: v.detach().clone() for k, v in ret[o].items() if torch.is_tensor(v)} for o in keep}
  assert ret["outputs_coarse_anchor"]["pts_traj_ref"].shape[0] > 0
  return ret, supervision(batch, cfg, dev)


def leaves(ret, dtype=torch.float32, device=DEV):
  """A copy of the output dicts whose differentiable entries are fresh leaves."""
  out = {}
  for o, d in ret.items():
    out[o] = {}
    for k, v in d.items():
      v = v.detach().to(device)
      if v.is_floating_point():
        v = v.to(dtype).clone()
        if k in GRAD_KEYS.get(o, ()):
          v.requires_grad_(True)
      out[o][k] = v
  return out


def variant(ret, rb, case):
  ret, rb = copy.copy({o: dict(d) for o, d in ret.items()}), dict(rb)
  ref, anc = ret["outputs_coarse_ref"], ret["outputs_coarse_anchor"]
  if case == "K0":
    for k in ("pts_traj_ref", "pts_traj_anchor"):
      anc[k] = anc[k][:0]
  elif case == "masked":
    for d in ret.values():
      d["mask"] = torch.zeros_like(d["mask"])
  elif case == "near":
    ref["depth"] = ref["depth"].clone()
    ref["depth"][:5] = torch.tensor([5e-3, 9.9e-3, 1e-4, 0.0, 2e-2], device=ref["depth"].device)
  elif case == "static_dy":  # rays the decomposition calls static with > 0.9 probability
    ref["weights_dy"] = ref["weights_dy"].clone()
    ref["weights_dy"][::2] *= 0.02
  return ret, rb


CASES = [("plain", 0), ("plain", INIT_DECAY + 50), ("static_dy", 5 * INIT_DECAY + 1), ("K0", 10), ("masked", 10),
         ("near", 2 * INIT_DECAY)]


def _both(rendered, case, epoch):
  from dynibar_b200 import criterion as cr
  ret, rb = variant(*rendered, case)
  args = loss_args()
  got_in = leaves(ret)
  table = cr.mono_step_table(got_in, rb, args, epoch)
  table[0].backward()
  want_in = leaves(ret, torch.float64, "cpu")
  rb64 = {k: v.cpu().double() for k, v in rb.items()}
  want, want_terms = loss_ref.mono_step_loss(want_in, rb64, args, epoch)
  want.backward()
  return cr, table.detach().cpu().double(), got_in, want_terms, want_in


@pytest.mark.parametrize("case,epoch", CASES)
def test_components_and_total_match_the_float64_restatement(rendered, case, epoch):
  cr, table, _, want, _ = _both(rendered, case, epoch)
  assert torch.isfinite(table).all()
  for i, name in enumerate(cr.TERM_NAMES):
    torch.testing.assert_close(table[i], want[name], rtol=2e-5, atol=1e-12, msg=lambda m: "%s: %s" % (name, m))
  divisor = epoch // INIT_DECAY
  if case == "static_dy":
    assert divisor > 4 and table[cr.COMPONENTS + cr.STATIC_DY] > 0  # the extra term is really there
  else:
    assert table[cr.COMPONENTS + cr.STATIC_DY] == 0
  assert (table[cr.COMPONENTS + cr.RGB_DYNAMIC] > 0) == (epoch < INIT_DECAY and case != "masked")
  if case == "K0":
    assert want["cycle_loss"] == 0 and table[7] == 0
  if case == "masked":  # every masked denominator on its epsilon
    for name in ("rgb_loss", "disp_loss", "flow_loss", "static_loss"):
      assert table[cr.TERM_NAMES.index(name)] == 0, name


@pytest.mark.parametrize("case,epoch", CASES)
def test_gradients_match_autograd_through_the_float64_restatement(rendered, case, epoch):
  _, _, got_in, _, want_in = _both(rendered, case, epoch)
  for o, keys in GRAD_KEYS.items():
    for k in keys:
      g, w = got_in[o][k].grad, want_in[o][k].grad
      if w is None or (w.numel() == 0):  # a term that is absent at this epoch, or K = 0
        assert g is None or g.numel() == 0, (o, k)
        continue
      assert g is not None and torch.isfinite(g).all(), (o, k)
      torch.testing.assert_close(g.cpu().double(), w, rtol=2e-4, atol=1e-6 * w.abs().max().item() + 1e-30,
                                 msg=lambda m: "%s/%s: %s" % (o, k, m))
  for o, keys in NO_GRAD_KEYS.items():
    for k in keys:
      assert got_in[o][k].grad is None, (o, k)
  ref = got_in["outputs_coarse_ref"]
  if epoch >= INIT_DECAY:
    assert ref["rgb_dy"].grad is None
  if case == "masked":
    for o, k in (("outputs_coarse_ref", "rgb"), ("outputs_coarse_ref", "rgb_static"), ("outputs_coarse_ref", "depth"),
                 ("outputs_coarse_ref", "render_flows"), ("outputs_coarse_anchor", "rgb")):
      assert (got_in[o][k].grad == 0).all(), (o, k)
  if case == "near":  # clamp active: no disparity gradient (rays 0-3), and one beside them that has it
    assert (ref["depth"].grad[:4] == 0).all()
    assert ref["depth"].grad[4] != 0 or not bool(ref["mask"][4])


def test_same_inputs_give_the_same_bits(rendered):
  from dynibar_b200 import criterion as cr
  ret, rb = variant(*rendered, "static_dy")
  runs = []
  for _ in range(2):
    x = leaves(ret)
    table = cr.mono_step_table(x, rb, loss_args(), 5 * INIT_DECAY)
    table[0].backward()
    runs.append([table.detach()] + [x[o][k].grad for o, ks in GRAD_KEYS.items() for k in ks if x[o][k].grad is not None])
  assert len(runs[0]) == len(runs[1]) > 10
  for a, b in zip(*runs):
    assert torch.equal(a, b)


def test_single_term_functions_are_the_fused_components(rendered):
  from dynibar_b200 import criterion as cr
  ret, rb = rendered
  x = leaves(ret)
  ref, ref_dy = x["outputs_coarse_ref"], x["outputs_coarse_ref_dy"]
  anc, anc_dy = x["outputs_coarse_anchor"], x["outputs_coarse_anchor_dy"]
  comp = cr.mono_step_table(x, rb, loss_args(), 0).detach()[cr.COMPONENTS:]
  mm = rb["motion_mask"]
  s = ref["s_vals"]
  crit = cr.Criterion()
  singles = {
      cr.RGB_REF: crit(ref, rb), cr.RGB_ANCHOR: cr.compute_temporal_rgb_loss(anc, rb),
      cr.RGB_DYNAMIC: cr.compute_rgb_loss(ref["rgb_dy"], rb, ref["mask"].float() * mm),
      cr.RGB_REF_DY: crit(ref_dy, rb, motion_mask=mm),
      cr.RGB_ANCHOR_DY: cr.compute_temporal_rgb_loss(anc_dy, rb, motion_mask=mm),
      cr.FLOW: cr.compute_flow_loss(ref["render_flows"], rb["flows"], ref["mask"].float()[None, :, None] * rb["masks"]),
      cr.DISTORTION: cr.eff_distloss_native(ref["weights"][:, :-1], (s[:, 1:] + s[:, :-1]) * 0.5,
                                            s[:, 1:] - s[:, :-1]),
  }
  for k, v in singles.items():
    assert v.dim() == 0 and v.requires_grad and torch.equal(v.detach(), comp[k]), (k, v.item(), comp[k].item())
  # each is differentiable on its own, with the fused call's gradient of that term
  for k in ("rgb", "weights"):
    ref[k].grad = None
  (singles[cr.RGB_REF] + singles[cr.DISTORTION]).backward()
  y = leaves(ret)
  want = loss_ref.criterion_rgb(y["outputs_coarse_ref"], rb) + loss_ref.distortion(
      y["outputs_coarse_ref"]["weights"][:, :-1], (s[:, 1:] + s[:, :-1]) * 0.5, s[:, 1:] - s[:, :-1])
  want.backward()
  for k in ("rgb", "weights"):
    torch.testing.assert_close(ref[k].grad, y["outputs_coarse_ref"][k].grad, rtol=2e-4,
                               atol=1e-5 * y["outputs_coarse_ref"][k].grad.abs().max().item())
  # warm-up loss == compute_rgb_loss on the same mask
  boot = cr.static_bootstrap_loss(x, rb)
  mask = (1.0 - rb["static_mask"]) * ref["mask"].float()
  assert torch.equal(boot, cr.compute_rgb_loss(x["outputs_coarse_st"]["rgb"], rb, mask))
  torch.testing.assert_close(boot.detach().cpu().double(),
                             loss_ref.static_bootstrap_loss(leaves(ret, torch.float64, "cpu"),
                                                            {k: v.cpu().double() for k, v in rb.items()}),
                             rtol=2e-5, atol=0.0)


def test_whole_training_step_matches_the_torch_loss_on_the_same_outputs():
  """render_rays_mono -> mono_step_loss -> backward() against the same step with the torch restatement of the loss
  applied to the same outputs (fp32 on the device): .grad of every parameter of the three networks, the three feature
  maps and trajectory_basis, at the bars of test_train_gpu.py."""
  from dynibar_b200 import criterion as cr, render_ray as rr
  from dynibar_b200.projection import Projector
  from test_train_gpu import _close
  cfg = dict(scenes.GOLDEN_CONFIGS["mono_train"])
  batch, feat_c, _, frame, t, offs, model, args = scenes.build(cfg)
  with torch.no_grad():
    model.motion_mlp.coeff_linear.weight.normal_(0.0, 0.05)
  dev = torch.device(DEV)
  m_dev = synthetic.model_to(model, dev)
  mods = {k: getattr(m_dev, k) for k in ("net_coarse_dy", "net_coarse_st", "motion_mlp")}
  for mod in mods.values():
    mod.requires_grad_(True)
  m_dev.trajectory_basis = m_dev.trajectory_basis.detach().requires_grad_(True)
  fd = tuple(f.to(dev).requires_grad_(True) for f in feat_c)
  rb = dict(synthetic.to_device(batch, dev), **supervision(batch, cfg, dev))
  largs = loss_args(args)

  def step(loss_fn):  # one forward + backward; the renderer's backward frees what it saved, so each loss renders anew
    ret = rr.render_rays_mono(frame, t, offs, rb, m_dev, fd, Projector(dev), cfg["N_samples"], largs, inv_uniform=True,
                              det=True, is_train=True, num_vv=cfg["num_vv"], precision="fp32")
    loss, terms = loss_fn(ret, rb, largs, 0)
    assert loss.dim() == 0 and loss.grad_fn is not None
    loss.backward()
    named = [("%s.%s" % (m, k), p) for m, mod in mods.items() for k, p in mod.named_parameters()]
    named += [("featmaps[%d]" % i, f) for i, f in enumerate(fd)] + [("trajectory_basis", m_dev.trajectory_basis)]
    grads = {}
    for k, p in named:
      assert p.grad is not None, k
      grads[k] = p.grad.clone()
      p.grad = None
    return terms, grads

  terms, got = step(cr.mono_step_loss)
  assert all(v.dim() == 0 and v.is_cuda and not v.requires_grad for v in terms.values())
  want_terms, want = step(loss_ref.mono_step_loss)
  for k in cr.TERM_NAMES:
    torch.testing.assert_close(terms[k], want_terms[k], rtol=1e-4, atol=1e-7, msg=lambda m: "%s: %s" % (k, m))
  for k, w in want.items():
    if k == "net_coarse_st.s":  # ill-conditioned on this rig, see test_train_gpu.py
      assert torch.isfinite(got[k]).all()
      continue
    assert w.abs().max() > 0, k
    _close(k, got[k], w.cpu(), 5e-3 if w.dim() > 1 else 2e-2)


# ---- the criterion at the training shape ------------------------------------------------------------------------
# Generated inputs (no renderer) with the keys and shapes render_rays_mono(is_train=True) and supervision() produce,
# at the reference's training batch (N_rand = 3072, N_samples = 64) and around every chunk and block edge of
# csrc/loss.cu: the distortion scan's 32-sample chunks (dist_n = S - 1 up to its limit of 256), the 8-ray blocks, the
# second pass over cdiv(R, 8) partial rows, and the K / n_sf lane loops.  Everything the kernels write is compared
# element by element with the float64 restatement under the bar of tests/geometry_stage_ref.py,
#     |got - ref| <= atol + ulps * (ulp(ref) + 2^-24 mag),
# mag being the sum of the absolute values of the terms the kernel adds times the length of its longest fp32 addition
# chain, plus the fp32 error of the ray's weights ratio rho where an output depends on it.  Kinks are kept out of the
# data rather than flagged: values on a 1/256 grid make every L1 difference exact (a tie is an exact 0 on both sides),
# rho stays clear of the 0.1 switch and of 1 - rho ~ 0, and depths clear of the 1e-2 clamp.
#
# ulps per output: 2x the worst measured (err - atol) / (ulp + 2^-24 mag) over every case below on an NVIDIA H100 80GB
# HBM3 (SXM) at its 700 W power limit; the worst value and its case are beside each.  atol is the smallest normal fp32
# number, so an exact zero passes against a reference that is zero.
TOL = {
    "components": (2.0 ** -126, 0.1),      # the 15 unweighted components; worst 0.0497 (S34)
    "totals": (2.0 ** -126, 0.067),        # the nine logged scalars; worst 0.0334 (S33)
    "g_rgb": (2.0 ** -126, 0.16),          # d rgb of the six rgb terms; worst 0.0753 (S34)
    "g_depth": (2.0 ** -126, 0.12),        # worst 0.0586 (S32)
    "g_flows": (2.0 ** -126, 0.05),        # worst 0.0248 (S34)
    "g_traj": (2.0 ** -126, 0.11),         # pts_traj_ref, pts_traj_anchor; worst 0.0521 (R8)
    "g_sf_seq": (2.0 ** -126, 0.48),       # worst 0.239 (S257)
    "g_weights": (2.0 ** -126, 0.24),      # the distortion scan backward; worst 0.120 (S32)
    "g_weights_dy": (2.0 ** -126, 0.121),  # entropy + static_dy; worst 0.0604 (S34)
    "g_weights_st": (2.0 ** -126, 0.017),  # entropy; worst 0.00802 (S32)
    "distloss": (2.0 ** -126, 0.087),      # eff_distloss_native; worst 0.0430 (n = 63)
    "g_distloss": (2.0 ** -126, 0.26),     # worst 0.128 (n = 64)
}
N_SF, N_FLOW = 6, 6


def _grid(g, shape, k=512):
  """Values j / 256, |j| <= k: exact in fp32, so every difference of two of them is exact."""
  return torch.randint(-k, k + 1, shape, generator=g).float() / 256.0


def _composited(g, R, S):
  """Alpha-compositing weights of random densities: each ray's sum is at most 1."""
  sigma = torch.rand(R, S, generator=g, dtype=torch.float64) * (6.0 / S) * torch.rand(R, 1, generator=g,
                                                                                    dtype=torch.float64)
  alpha = 1.0 - torch.exp(-sigma)
  T = torch.cumprod(torch.cat([torch.ones(R, 1, dtype=torch.float64), 1.0 - alpha[:, :-1]], -1), -1)
  return alpha * T


def generated(R, S, K, seed, zero_masks=False):
  """(output dicts, supervision) of one training step, seeded, on the CPU in fp32."""
  g = torch.Generator().manual_seed(seed)
  rand = lambda *s: torch.rand(*s, generator=g)
  bits = lambda *s: rand(*s) > 0.5
  # weights_dy / weights_st with the ray's ratio rho drawn in [0.01, 0.95] outside [0.09, 0.11]; then a ray of every
  # 16 with both zero (the 1e-9 clamp), one with no static weight (rho = 1) and one with no dynamic weight (rho = 0)
  wd, ws = _composited(g, R, S), _composited(g, R, S)
  rho = 0.01 + 0.94 * torch.rand(R, generator=g, dtype=torch.float64)
  rho = torch.where((rho - 0.1).abs() < 0.01, rho + 0.03, rho)
  a, b = wd.sum(-1), ws.sum(-1)
  k = rho * b / ((1.0 - rho) * a)
  wd = torch.where(k[:, None] <= 1.0, wd * k[:, None], wd)
  ws = torch.where(k[:, None] > 1.0, ws / k[:, None], ws)
  wd[1::16], ws[1::16], ws[2::16], wd[3::16] = 0.0, 0.0, 0.0, 0.0
  near = 0.5 + rand(R, 1)
  far = near * (4.0 + 20.0 * rand(R, 1))
  t = torch.sort(torch.cat([torch.zeros(R, 1), rand(R, S - 2), torch.ones(R, 1)], -1), -1).values
  s_vals = 1.0 / (1.0 / near * (1.0 - t) + 1.0 / far * t)  # inverse-uniform: increasing in t
  s_vals = torch.sort(s_vals, -1).values
  occ = rand(R, S)
  u = rand(R, S)
  occ[u < 0.1], occ[u > 0.9] = 0.0, 1.0
  depth = 0.05 + 10.0 * rand(R)
  depth[:4] = torch.tensor([5e-3, 9.9e-3, 1e-4, 0.0])[:R]
  gt_disp = 1.0 / depth.clamp(min=1e-2) + torch.where(bits(R), 1.0, -1.0) * (1e-3 + rand(R))
  traj_ref = _grid(g, (K, R, S, 3))
  traj_anchor = torch.where(rand(K, R, S, 3) < 0.1, traj_ref, _grid(g, (K, R, S, 3)))
  mask = lambda: torch.zeros(R, dtype=torch.bool) if zero_masks else bits(R)
  ref = {"rgb": rand(R, 3), "rgb_dy": rand(R, 3), "rgb_static": rand(R, 3), "depth": depth,
         "render_flows": _grid(g, (N_FLOW, R, 2)), "weights": _composited(g, R, S).float(), "weights_dy": wd.float(),
         "weights_st": ws.float(), "mask": mask(), "s_vals": s_vals}
  anc = {"rgb": rand(R, 3), "mask": mask(), "occ_weight_map": rand(R), "pts_traj_ref": traj_ref,
         "pts_traj_anchor": traj_anchor, "occ_weights": occ, "sf_seq": _grid(g, (N_SF, R, S, 3), 256)}
  ret = {"outputs_coarse_ref": ref, "outputs_coarse_ref_dy": {"rgb": rand(R, 3), "mask": mask()},
         "outputs_coarse_anchor": anc,
         "outputs_coarse_anchor_dy": {"rgb": rand(R, 3), "mask": mask(), "occ_weight_map": rand(R)}}
  motion = torch.zeros(R) if zero_masks else bits(R).float()
  flow_masks = torch.zeros(N_FLOW, R, 1) if zero_masks else bits(N_FLOW, R, 1).float()
  rb = {"rgb": rand(R, 3), "disp": gt_disp, "motion_mask": motion, "static_mask": bits(R).float(),
        "flows": torch.where(rand(N_FLOW, R, 2) < 0.1, ref["render_flows"], _grid(g, (N_FLOW, R, 2))),
        "masks": flow_masks}
  return ret, rb


def ref_components(ret, rb, args, epoch):
  """term index -> the float64 component (the term before its weight) from loss_ref's helpers."""
  from dynibar_b200 import criterion as cr
  ref, ref_dy = ret["outputs_coarse_ref"], ret["outputs_coarse_ref_dy"]
  anc, anc_dy = ret["outputs_coarse_anchor"], ret["outputs_coarse_anchor_dy"]
  sw = loss_ref.step_weights(args, epoch)
  motion, pred_mask = rb["motion_mask"], ref["mask"].double()
  zero = torch.zeros((), dtype=torch.float64)
  sum_dy, sum_st = ref["weights_dy"].sum(-1), ref["weights_st"].sum(-1)
  ratio = sum_dy / torch.clamp(sum_dy + sum_st, min=1e-9)
  smask = (1.0 - rb["static_mask"]) * pred_mask * (1.0 - ratio)
  m2 = smask * (ratio < 0.1).double()
  t_ref, t_anc = anc["pts_traj_ref"], anc["pts_traj_anchor"]
  occ = anc["occ_weights"][None, ..., None].expand(t_anc.shape[0], -1, -1, 3)
  sf, s = anc["sf_seq"], ref["s_vals"]
  return {
      cr.RGB_REF: loss_ref.criterion_rgb(ref, rb), cr.RGB_ANCHOR: loss_ref.temporal_rgb(anc, rb),
      cr.RGB_DYNAMIC: loss_ref.rgb_loss(ref["rgb_dy"], rb, pred_mask * motion) if sw["dynamic_rgb"] else zero,
      cr.RGB_REF_DY: loss_ref.criterion_rgb(ref_dy, rb, motion_mask=motion),
      cr.RGB_ANCHOR_DY: loss_ref.temporal_rgb(anc_dy, rb, motion_mask=motion),
      cr.STATIC: loss_ref.rgb_loss(ref["rgb_static"], rb, smask),
      cr.DISP: ((1.0 / ref["depth"].clamp(min=1e-2) - rb["disp"]).abs() * pred_mask).sum() / (pred_mask.sum() + 1e-8),
      cr.FLOW: loss_ref.flow_l1(ref["render_flows"], rb["flows"], pred_mask[None, :, None] * rb["masks"]),
      cr.CYCLE: ((t_ref - t_anc).abs() * occ).sum() / (occ.sum() + 1e-8),
      cr.REG_ABS: sf.abs().mean(), cr.REG_TIME: ((sf[:-1] - sf[1:]) ** 2).mean(),
      cr.REG_SPACE: (sf[:, :, 1:] - sf[:, :, :-1]).abs().mean(),
      cr.ENTROPY: (-(ratio * torch.log(ratio + 1e-9) + (1.0 - ratio) * torch.log(1.0 - ratio + 1e-9))).mean(),
      cr.DISTORTION: loss_ref.distortion(ref["weights"][:, :-1], (s[:, 1:] + s[:, :-1]) * 0.5, s[:, 1:] - s[:, :-1]),
      cr.STATIC_DY: (sum_dy * m2).abs().sum() / (m2 + 1e-8).sum() if sw["static_dy"] else zero,
  }


def _chunks(n):
  """Longest fp32 addition chain of a warp's sum of n elements: n / 32 per lane, then the 5-level shuffle tree."""
  return -(-n // 32) + 5


def dist_mags(w, m, iv):
  """float64 [R,n] -> (forward, backward) magnitudes of the distortion scan per sample: the sums of the absolute
  values of the prefix-sum terms the kernel adds and cancels, times the scan's chain length."""
  W, WM = torch.cumsum(w, -1), torch.cumsum(w * m, -1)
  exW, exWM = W - w, WM - w * m
  L = _chunks(w.shape[-1])
  fwd = (2.0 * w * (m * exW + exWM) * L + iv * w * w / 3.0)
  bwd = 2.0 * (m * exW + exWM + (WM[:, -1:] + WM) + m * (W[:, -1:] + W)) * L + (2.0 / 3.0) * iv * w
  return fwd, bwd


def entropy_mags(sum_dy, sum_st, L):
  """Per-ray magnitudes of the entropy term: of its value, and of d value / d weights_dy and d weights_st, including the
  fp32 error of rho (2 L 2^-24 rho through the ray sums)."""
  c = torch.clamp(sum_dy + sum_st, min=1e-9)
  rho = sum_dy / c
  p, q = rho + 1e-9, 1.0 - rho + 1e-9
  d_rho = 2.0 * L * rho * (1.0 / p + 1.0 / q)  # |d dv / d rho| * (rho error / 2^-24)
  dv = torch.log(p).abs() + rho / p + torch.log(q).abs() + (1.0 - rho) / q + d_rho
  v = -(rho * torch.log(p) + (1.0 - rho) * torch.log(q)) * L + 2.0 * L * rho * (torch.log(q / p)).abs()
  return v, dv * (1.0 / c + sum_dy / c ** 2), rho


def _check(name, got, ref, mag, worst):
  """Assert got within the bar of TOL[name's group] everywhere; record the group's worst excess in `worst`."""
  got, ref, mag = got.detach().cpu().double(), ref.detach().double(), mag.double()
  assert torch.isfinite(got).all(), name
  key = name.split("/")[0]
  x = excess(key, got, ref, mag, 0.0, tol=TOL)
  worst[key] = max(worst.get(key, -math.inf), x.max().item())
  bad = (got - ref).abs() > bar(key, ref, mag, 0.0, tol=TOL)
  assert not bad.any(), "%s: %d of %d over the bar; worst excess %.3g ulps (bar %.3g), at %s: got %r want %r" % (
      name, int(bad.sum()), bad.numel(), x.max().item(), TOL[key][1], tuple(bad.nonzero()[0].tolist()),
      got[bad][0].item(), ref[bad][0].item())


def _poison_allocator():
  """Fill freed blocks of both pools of the caching allocator with NaN.  This makes it likely, not certain, that a
  gradient element the backward kernel fails to write reads as NaN rather than a stale 0; the guard that does not
  depend on the allocator is the exact-0 check of the last weight column."""
  blocks = [torch.full((255 << 10,), math.nan, device=DEV) for _ in range(32)]
  blocks.append(torch.full((64 << 20,), math.nan, device=DEV))
  del blocks


def _report(tag, worst):
  print("\n[%s] worst excess (ulps): %s" % (tag, ", ".join("%s %.3g" % kv for kv in sorted(worst.items()))))


def training_case(R, S, K, seed, epoch, zero_masks=False):
  """Run the criterion on generated inputs and compare everything it writes with the float64 restatement; returns
  the device table and the gradients (for the repeat test)."""
  from dynibar_b200 import criterion as cr
  ret, rb = generated(R, S, K, seed, zero_masks)
  args = loss_args()
  got_in = leaves(ret)
  rb_dev = {k: v.to(DEV) for k, v in rb.items()}
  table = cr.mono_step_table(got_in, rb_dev, args, epoch)
  _poison_allocator()
  table[0].backward()
  torch.cuda.synchronize()
  want_in = leaves(ret, torch.float64, "cpu")
  rb64 = {k: v.double() for k, v in rb.items()}
  want, want_terms = loss_ref.mono_step_loss(want_in, rb64, args, epoch)
  want.backward()
  got_t = table.detach().cpu().double()
  worst = {}
  # chain lengths: a ray's lane loops, the block's 8 rows and the second pass over cdiv(R, 8) rows.  Every gradient
  # is scaled by weight / denominator, and the denominators pass through the second pass, so L bounds the gradients
  # too; at R = 65536 (L ~ 8200) that makes the bars loose by construction, about 5e-4 relative x ulps.
  nblocks = -(-R // 8)
  L = _chunks(3 * S * max(K, N_SF)) + 8 + nblocks + 4
  Ls = _chunks(S) + 2
  with torch.no_grad():
    d = {o: {k: v.detach() for k, v in dd.items()} for o, dd in want_in.items()}
    ref, anc = d["outputs_coarse_ref"], d["outputs_coarse_anchor"]
    comp = ref_components(d, rb64, args, epoch)
    s = ref["s_vals"]
    w, m, iv = ref["weights"][:, :-1], (s[:, 1:] + s[:, :-1]) * 0.5, s[:, 1:] - s[:, :-1]
    fwd_d, bwd_d = dist_mags(w, m, iv)
    sum_dy, sum_st = ref["weights_dy"].sum(-1), ref["weights_st"].sum(-1)
    ent_v, ent_dv, rho = entropy_mags(sum_dy, sum_st, Ls)
    one_minus = torch.where(rho < 1.0, 2.0 * Ls * rho / (1.0 - rho), torch.zeros_like(rho))
    cmag = {k: L * v.abs() for k, v in comp.items()}
    cmag[cr.DISTORTION] = (L * comp[cr.DISTORTION].abs() * R + fwd_d.sum()) / R
    cmag[cr.ENTROPY] = (L * comp[cr.ENTROPY].abs() * R + ent_v.sum()) / R
    cmag[cr.STATIC] = (L + one_minus.max()) * comp[cr.STATIC].abs()
    wt = cr.step_weights(args, epoch)
    # which terms the step has, from the restatement's schedule (not the one under test)
    sw = loss_ref.step_weights(args, epoch)
    present = {k: True for k in range(15)}
    present[cr.RGB_DYNAMIC], present[cr.STATIC_DY], present[cr.CYCLE] = sw["dynamic_rgb"], sw["static_dy"], K > 0
    for k, v in comp.items():
      if not present[k]:
        assert got_t[cr.COMPONENTS + k] == 0, k
        continue
      _check("components/%d" % k, got_t[cr.COMPONENTS + k], v, cmag[k], worst)
    # the nine scalars are sums of weighted components
    tmag = {k: abs(wt.w[k]) * (cmag[k] + 4 * comp[k].abs()) if present[k] else torch.zeros(()) for k in comp}
    groups = {"loss": range(15), "flow_loss": [cr.FLOW], "disp_loss": [cr.DISP], "rgb_loss": range(5),
              "distortion_loss": [cr.DISTORTION], "entropy_loss": [cr.ENTROPY], "static_loss": [cr.STATIC, cr.STATIC_DY],
              "cycle_loss": [cr.CYCLE], "reg_loss": [cr.REG_ABS, cr.REG_TIME, cr.REG_SPACE]}
    for i, name in enumerate(cr.TERM_NAMES):
      _check("totals/" + name, got_t[i], want_terms[name], sum(tmag[k] for k in groups[name]) + 16 * want_terms[name].abs(),
             worst)
    # gradients
    g_ent = wt.w[cr.ENTROPY] / R
    for o, keys in GRAD_KEYS.items():
      for k in keys:
        gg, ww = got_in[o][k].grad, want_in[o][k].grad
        if ww is None or ww.numel() == 0:
          assert gg is None or gg.numel() == 0, (o, k)
          continue
        assert gg is not None, (o, k)
        mag = L * ww.abs()
        key = {"depth": "g_depth", "render_flows": "g_flows", "pts_traj_ref": "g_traj", "pts_traj_anchor": "g_traj",
               "sf_seq": "g_sf_seq", "weights": "g_weights", "weights_dy": "g_weights_dy",
               "weights_st": "g_weights_st"}.get(k, "g_rgb")
        if o == "outputs_coarse_ref" and k == "rgb_static":
          mag = mag + one_minus[:, None] * ww.abs()
        elif k == "weights":
          mag = mag + F.pad(abs(wt.w[cr.DISTORTION]) / R * bwd_d, (0, 1))
          # the last sample, which the distortion term does not read, gets exactly 0
          assert (gg[:, -1] == 0).all()
        elif k in ("weights_dy", "weights_st"):
          mag = mag + (abs(g_ent) * ent_dv)[:, None] * Ls + (abs(wt.w[cr.STATIC_DY]) / R)
        elif k == "sf_seq":
          x = anc["sf_seq"]
          s_abs, s_time = wt.w[cr.REG_ABS] / x.numel(), wt.w[cr.REG_TIME] / x[1:].numel()
          s_space = wt.w[cr.REG_SPACE] / x[:, :, 1:].numel()
          t_next = F.pad(2.0 * (x[:-1].abs() + x[1:].abs()), (0, 0, 0, 0, 0, 0, 0, 1))
          t_prev = F.pad(2.0 * (x[:-1].abs() + x[1:].abs()), (0, 0, 0, 0, 0, 0, 1, 0))
          mag = mag + 4.0 * (s_abs + s_time * (t_next + t_prev) + 2.0 * s_space)
        _check("%s/%s/%s" % (key, o, k), gg, ww, mag, worst)
  return table.detach(), [got_in[o][k].grad for o, ks in GRAD_KEYS.items() for k in ks
                          if got_in[o][k].grad is not None], worst


TRAINING_EPOCHS = (0, INIT_DECAY + 50, 5 * INIT_DECAY + 1)  # divisor 0, 1 and 5 (static_dy on)
SHAPES = ([("train", 3072, 64, 3, e) for e in TRAINING_EPOCHS] +
          [("S%d" % S, 96, S, 2, 5 * INIT_DECAY + 1 if S % 2 else 0) for S in (32, 33, 34, 64, 128, 257)] +
          [("R%d" % R, R, 64, 3, 10) for R in (1, 7, 8, 9, 3071, 3073)] +
          [("R65536", 65536, 8, 3, 5 * INIT_DECAY + 1)] +
          [("K%d" % K, 40, 64, K, 10) for K in (0, 1, 7)] +
          [("masked", 200, 64, 3, 10), ("masked_static_dy", 200, 34, 3, 5 * INIT_DECAY + 1)])


@pytest.mark.parametrize("tag,R,S,K,epoch", SHAPES, ids=["%s-e%d" % (s[0], s[4]) for s in SHAPES])
def test_criterion_at_training_shapes_matches_the_float64_restatement(tag, R, S, K, epoch):
  table, _, worst = training_case(R, S, K, 1000 + R + 7 * S + K, epoch, zero_masks=tag.startswith("masked"))
  _report("%s R=%d S=%d K=%d epoch=%d" % (tag, R, S, K, epoch), worst)
  if tag.startswith("masked"):
    from dynibar_b200 import criterion as cr
    for name in ("rgb_loss", "disp_loss", "flow_loss"):
      assert table[cr.TERM_NAMES.index(name)] == 0, name


def test_training_batch_gives_the_same_bits_on_a_repeat():
  runs = [training_case(3072, 64, 3, 77, 5 * INIT_DECAY + 1)[:2] for _ in range(2)]
  assert len(runs[0][1]) == len(runs[1][1]) > 10
  assert torch.equal(runs[0][0], runs[1][0])
  for a, b in zip(runs[0][1], runs[1][1]):
    assert torch.equal(a, b)


def _distloss_inputs(R, n, seed):
  g = torch.Generator().manual_seed(seed)
  w = _composited(g, R, n).float()
  s = torch.sort(torch.rand(R, n + 1, generator=g) * 10.0 + 0.5, -1).values
  return w, ((s[:, 1:] + s[:, :-1]) * 0.5), s[:, 1:] - s[:, :-1]


@pytest.mark.parametrize("n", [31, 32, 33, 63, 64, 256])
def test_eff_distloss_native_matches_the_pairwise_definition(n):
  from dynibar_b200 import criterion as cr
  R = 67
  w, m, iv = _distloss_inputs(R, n, 5 + n)
  x = w.to(DEV).requires_grad_(True)
  got = cr.eff_distloss_native(x, m.to(DEV), iv.to(DEV))
  _poison_allocator()
  got.backward()
  w64 = w.double().requires_grad_(True)
  want = loss_ref.distortion_pairwise(w64, m.double(), iv.double())
  want.backward()
  fwd, bwd = dist_mags(w.double(), m.double(), iv.double())
  L = _chunks(n) + 8 + -(-R // 8) + 4
  worst = {}
  _check("distloss", got, want, (L * want.abs() * R + fwd.sum()) / R, worst)
  _check("g_distloss", x.grad, w64.grad, L * w64.grad.abs() + bwd / R, worst)
  _report("eff_distloss_native n=%d" % n, worst)


def test_eff_distloss_native_refuses_more_than_256_samples():
  from dynibar_b200 import criterion as cr
  w, m, iv = (t.to(DEV) for t in _distloss_inputs(3, 257, 1))
  with pytest.raises(RuntimeError, match="at most 256 samples per ray, got 257"):
    cr.eff_distloss_native(w, m, iv)
