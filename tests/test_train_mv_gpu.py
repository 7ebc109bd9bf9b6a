"""Training of render_rays_mv's fine stage and of the trajectory bases (row f2) against torch autograd through the
oracle: the fine pass of render_rays_mv (fine_render_rays, render_ray.py:407-597) with its coarse pass under no_grad
(:672), trajectory_basis / trajectory_basis_fine as trainable tensors (ibrnet/model.py:94-118, :331-351), and the two
kernels that make them differentiable: the basis-row gradient of traj_combine and the expected scene flow
(:585-595).  Bars: those of test_train_gpu.py.

The fine-stage step at the Nvidia benchmark shape, with a stand-in loss, every gradient against a float64 reference at
per-tensor bars and planted glue errors, is tests/test_train_mv_step_gpu.py."""

import pytest
import torch

import scenes
from dynibar_b200 import synthetic
from oracle import dynibar_oracle as orc
from test_train_gpu import _TRAIN_KEYS, _close, _leaves

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

_MV_CASES = {
    "mv_small": dict(scenes.GOLDEN_CONFIGS["mv_small"], stress=False),
    "mv_linear": scenes.GOLDEN_CONFIGS["mv_linear"],
    # the Nvidia benchmark's view counts and sample counts (7 + 11 views, 64 + 64 samples), a few rays
    "mv_nvidia": dict(scenes.GOLDEN_CONFIGS["mv_small"], V_dy=7, V_st=11, N_samples=64, N_importance=64, rays=4,
                      stress=False, seed=21),
}
_FINE_KEYS = {
    "outputs_fine_ref": ("rgb", "rgb_static", "rgb_dy", "depth", "weights", "weights_dy", "weights_st", "alpha",
                         "alpha_dy", "render_flows", "exp_sf"),
    "outputs_fine_ref_dy": ("rgb", "depth", "weights"),
}
_FINE = ("net_fine_dy", "net_fine_st", "motion_mlp_fine")
_COARSE = ("net_coarse_dy", "net_coarse_st", "motion_mlp")


def _mv_scene(name, rays=None):
  cfg = dict(_MV_CASES[name])
  if rays is not None:
    cfg["rays"] = rays
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  with torch.no_grad():  # larger motion than the bench initialisation so that its gradients are well above rounding
    model.motion_mlp_fine.coeff_linear.weight.normal_(0.0, 0.05)
  return cfg, batch, feat_c, feat_f, frame, t, offs, model, args


def _mv_device(model, batch, feat_c, feat_f, basis_grad=True):
  dev = torch.device(DEV)
  m = synthetic.model_to(model, dev)
  for name in _FINE + _COARSE:  # coarse modules too: render_rays_mv must leave them without gradients
    getattr(m, name).requires_grad_(True)
  m.trajectory_basis_fine = m.trajectory_basis_fine.detach().requires_grad_(basis_grad)
  fc = tuple(f.to(dev).requires_grad_(True) if f is not None else None for f in feat_c)
  ff = tuple(f.to(dev).requires_grad_(True) if f is not None else None for f in feat_f)
  return m, synthetic.to_device(batch, dev), fc, ff


def _grad_tol(prec, mname, k, p):
  if prec == "fp32":
    return 5e-3 if p.dim() > 1 else 2e-2
  if mname.startswith("motion_mlp") and k.startswith("pts_linears"):
    return 2e-1  # ReLU kinks under bf16 rounding (test_train_gpu.py)
  return 5e-2 if p.dim() > 1 else 1.5e-1


@pytest.mark.parametrize("name,prec,rays", [("mv_small", "fp32", None), ("mv_linear", "fp32", None),
                                            ("mv_nvidia", "fp32", None), ("mv_small", "bf16", 96)])
def test_render_rays_mv_fine_stage_matches_oracle_autograd(name, prec, rays):
  """loss = randomly weighted fine outputs of render_rays_mv; d loss / d (every parameter of net_fine_dy, net_fine_st,
  motion_mlp_fine, trajectory_basis_fine, both fine feature maps) against torch autograd through the oracle."""
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  cfg, batch, feat_c, feat_f, frame, t, offs, model, args = _mv_scene(name, rays)
  kw = dict(inv_uniform=cfg["inv_uniform"], N_importance=cfg["N_importance"], det=True, is_train=True)
  g = torch.Generator().manual_seed(7)
  # ---- oracle (CPU): leaf copies of the fine stage
  om = type(model)(**vars(model))
  om.net_fine_dy = _leaves(model.net_fine_dy, model.net_fine_dy.shift)
  om.net_fine_st = _leaves(model.net_fine_st)
  om.motion_mlp_fine = _leaves(model.motion_mlp_fine)
  om.trajectory_basis_fine = model.trajectory_basis_fine.clone().requires_grad_(True)
  fo = tuple(f.clone().requires_grad_(True) if f is not None else None for f in feat_f)
  want = orc.render_rays_mv(frame, t, offs, batch, om, None, feat_c, fo, cfg["N_samples"], args, **kw)
  gens = {(o, k): torch.randn(want[o][k].shape, generator=g) for o, ks in _FINE_KEYS.items() for k in ks}
  sum((want[o][k] * v).sum() for (o, k), v in gens.items()).backward()
  # ---- library (GPU)
  m, b, fc, ff = _mv_device(model, batch, feat_c, feat_f)
  with torch.no_grad():
    plain = rr.render_rays_mv(frame, t, offs, b, m, Projector(DEV), fc, ff, cfg["N_samples"], args, precision=prec,
                              **kw)
  got = rr.render_rays_mv(frame, t, offs, b, m, Projector(DEV), fc, ff, cfg["N_samples"], args, precision=prec, **kw)
  assert got["outputs_fine_anchor"] is None and got["outputs_fine_anchor_dy"] is None
  # the coarse pass and the resampled depths are the forward path's, bit for bit
  for k, v in plain["outputs_coarse_ref"].items():
    assert not got["outputs_coarse_ref"][k].requires_grad, k
    assert torch.equal(got["outputs_coarse_ref"][k], v), k
  for k in ("z_vals", "s_vals"):
    assert torch.equal(got["outputs_fine_ref"][k], plain["outputs_fine_ref"][k]), k
  assert list(got["outputs_fine_ref"].keys()) == list(plain["outputs_fine_ref"].keys())
  ft = dict(rtol=1e-3, atol=2e-4) if prec == "fp32" else dict(rtol=3e-2, atol=2e-2)
  for (o, k), v in gens.items():
    assert got[o][k].requires_grad, (o, k)
    if k == "render_flows":  # pixels: compare relative to their scale
      ft_k = dict(rtol=1e-3, atol=1e-2) if prec == "fp32" else None
    else:
      ft_k = ft
    if ft_k is not None:
      torch.testing.assert_close(got[o][k].detach().cpu(), want[o][k].detach(),
                                 msg=lambda s: "%s/%s: %s" % (o, k, s), **ft_k)
  sum((got[o][k] * v.to(DEV)).sum() for (o, k), v in gens.items()).backward()
  for mname in _FINE:
    w = getattr(om, mname)
    for k, p in getattr(m, mname).named_parameters():
      assert p.grad is not None, (mname, k)
      if mname == "net_fine_st" and k == "s":  # ill-conditioned (test_train_gpu.py)
        assert torch.isfinite(p.grad).all()
        continue
      _close("%s.%s" % (mname, k), p.grad, w[k].grad, _grad_tol(prec, mname, k, p), floor=1e-5)
  _close("trajectory_basis_fine", m.trajectory_basis_fine.grad, om.trajectory_basis_fine.grad,
         5e-3 if prec == "fp32" else 5e-2, floor=1e-6)
  for i in (0, 2):
    _close("fine_featmaps[%d]" % i, ff[i].grad, fo[i].grad, 5e-3 if prec == "fp32" else 5e-2)
  # the coarse stage never trains (render_ray.py:672)
  for mname in _COARSE:
    assert all(p.grad is None for p in getattr(m, mname).parameters()), mname
  assert all(f.grad is None for f in fc if f is not None)


def _mono_scene(name, prec):
  if name != "mono_wrap":
    cfg = dict(scenes.GOLDEN_CONFIGS[name])
    if prec == "bf16":
      cfg["rays"] = 96  # >= 2048 (point, view) rows per product: the tensor-core kernels take over
    return (cfg,) + tuple(scenes.build(cfg))
  # reference frame 1: rows f - 2 and f - 3 of the basis wrap to the last frames, as in the reference
  cfg = dict(scenes.GOLDEN_CONFIGS["mono_train"], seed=16)
  batch, feat_c, feat_f, frame, t, offs = synthetic.make_scene(
      H=cfg["H"], W=cfg["W"], V_dy=cfg["V_dy"], V_st=cfg["V_st"], num_vv=cfg["num_vv"], seed=cfg["seed"],
      rays=cfg["rays"], frame_idx=1, anchor_offset=cfg["anchor_offset"])
  args = synthetic.make_args(cfg["anti_alias_pooling"], cfg["mask_rgb"], cfg["occ_weights_mode"])
  model, args = synthetic.make_model(cfg["N_samples"], 0, args=args, seed=cfg["seed"], mono=True)
  return cfg, batch, feat_c, feat_f, frame, t, offs, model, args


@pytest.mark.parametrize("name,prec", [("mono_train", "fp32"), ("mono_train_near", "fp32"), ("mono_wrap", "fp32"),
                                       ("mono_train", "bf16")])
def test_render_rays_mono_basis_gradient_matches_oracle_autograd(name, prec):
  """render_rays_mono(is_train=True) with trajectory_basis requiring grad: d loss / d basis through every displaced
  point (seq, sf_seq, pts_anchor and the second MotionMLP call, seq_a, pts_traj_ref) against oracle autograd; the
  forward outputs are those of the same call with the basis frozen, bit for bit."""
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  cfg, batch, feat_c, _, frame, t, offs, model, args = _mono_scene(name, prec)
  with torch.no_grad():
    model.motion_mlp.coeff_linear.weight.normal_(0.0, 0.05)
  kw = dict(inv_uniform=cfg["inv_uniform"], det=True, is_train=True, num_vv=cfg["num_vv"])
  g = torch.Generator().manual_seed(31)
  om = type(model)(**vars(model))
  om.net_coarse_dy = _leaves(model.net_coarse_dy, model.net_coarse_dy.shift)
  om.net_coarse_st = _leaves(model.net_coarse_st)
  om.motion_mlp = _leaves(model.motion_mlp)
  om.trajectory_basis = model.trajectory_basis.clone().requires_grad_(True)
  want = orc.render_rays_mono(frame, t, offs, batch, om, feat_c, None, cfg["N_samples"], args, **kw)
  gens = {(o, k): torch.randn(want[o][k].shape, generator=g) for o, ks in _TRAIN_KEYS.items() for k in ks}
  sum((want[o][k] * v).sum() for (o, k), v in gens.items()).backward()
  dev = torch.device(DEV)
  m = synthetic.model_to(model, dev)
  for name_ in _COARSE:
    getattr(m, name_).requires_grad_(True)
  b = synthetic.to_device(batch, dev)
  fd = tuple(f.to(dev) for f in feat_c)
  frozen = rr.render_rays_mono(frame, t, offs, b, m, fd, Projector(dev), cfg["N_samples"], args, precision=prec, **kw)
  m.trajectory_basis = m.trajectory_basis.detach().requires_grad_(True)
  got = rr.render_rays_mono(frame, t, offs, b, m, fd, Projector(dev), cfg["N_samples"], args, precision=prec, **kw)
  for o, part in frozen.items():
    if part is None:
      assert got[o] is None
      continue
    for k, v in part.items():
      assert torch.equal(got[o][k], v), (o, k)
  sum((got[o][k] * v.to(dev)).sum() for (o, k), v in gens.items()).backward()
  _close("trajectory_basis", m.trajectory_basis.grad, om.trajectory_basis.grad, 5e-3 if prec == "fp32" else 5e-2,
         floor=1e-6)


@pytest.mark.parametrize("n,nb,P", [(1, 1, 1), (3, 8, 1023), (7, 6, 3077), (16, 8, 5000), (12, 5, 1024 * 3),
                                    (16, 6, 196608)])
def test_traj_combine_basis_gradient_matches_fp64(n, nb, P):
  """gD[i,k] = sum_p sum_a g[i,p,a] coeff[p,a nb+k]: against an fp64 reduction, P not a multiple of the block, and the
  same bits on a second call (no float atomics)."""
  from dynibar_b200 import autograd as ag
  g = torch.Generator().manual_seed(n * 100 + nb + P)
  coeff = torch.randn(1, P, 3 * nb, generator=g)
  D = torch.randn(n, nb, generator=g)
  gout = torch.randn(n, 1, P, 3, generator=g)
  want = torch.einsum("ipa,pak->ik", gout[:, 0].double(), coeff[0].double().reshape(P, 3, nb))
  scale = torch.einsum("ipa,pak->ik", gout[:, 0].double().abs(), coeff[0].double().abs().reshape(P, 3, nb))
  grads = []
  for _ in range(2):
    Dd = D.to(DEV).requires_grad_(True)
    out = ag.traj_combine(coeff.to(DEV), Dd)
    out.backward(gout.to(DEV))
    grads.append(Dd.grad.clone())
  assert torch.equal(grads[0], grads[1])
  err = (grads[0].cpu().double() - want).abs()
  assert (err <= 1e-5 * scale + 1e-6).all(), err.max().item()


def test_expected_scene_flow_matches_torch_max():
  """exp_sf = max(sum_s w sf[0], sum_s w sf[1]) forward and backward against torch autograd of torch.max(p, m),
  including exact ties: rays whose motion coefficients are all zero (the reference's zero-initialised coeff_linear,
  or samples in the zeroed last 10 %) have both sums exactly 0."""
  from dynibar_b200 import autograd as ag, synthetic as syn
  g = torch.Generator().manual_seed(3)
  R, S, nb = 37, 128, 6
  w = torch.softmax(torch.randn(R, S, generator=g), 1)
  coeff = torch.randn(R, S, 3 * nb, generator=g) * 0.1
  coeff[:9] = 0.0                                    # ties everywhere on these rays
  basis = syn.init_dct_basis(nb, 24)
  D = torch.stack([basis[12] - basis[10], basis[8] - basis[10]])
  sf = ag.traj_combine(coeff.to(DEV), D.to(DEV)).cpu()
  assert (sf[:, :9] == 0).all()
  sf[1, 9:12] = sf[0, 9:12]                          # equal halves: ties with non-zero sums
  gout = torch.randn(R, 3, generator=g)
  wo, so = w.double().requires_grad_(True), sf.double().requires_grad_(True)
  p = (wo[..., None] * so[0]).sum(1)
  mm = (wo[..., None] * so[1]).sum(1)
  want = torch.max(p, mm)
  (want * gout.double()).sum().backward()
  wd, sd = w.to(DEV).requires_grad_(True), sf.to(DEV).requires_grad_(True)
  got = ag.expected_scene_flow(wd, sd)
  torch.testing.assert_close(got.detach().cpu().double(), want.detach(), rtol=1e-5, atol=1e-6)
  (got * gout.to(DEV)).sum().backward()
  torch.testing.assert_close(wd.grad.cpu().double(), wo.grad, rtol=1e-5, atol=1e-6)
  torch.testing.assert_close(sd.grad.cpu().double(), so.grad, rtol=1e-5, atol=1e-6)
  # the tie rule itself: half of the gradient to each side
  torch.testing.assert_close(sd.grad[0, :12].cpu(), sd.grad[1, :12].cpu(), rtol=0, atol=0)
  torch.testing.assert_close(sd.grad[0, :9].cpu(), 0.5 * w[:9, :, None] * gout[:9, None, :], rtol=1e-6, atol=1e-7)


def test_mv_training_ray_slices_match_one_call(monkeypatch):
  """A small TRAIN_ROWS_LIMIT renders the fine stage in slices: same outputs and gradients as one call."""
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  cfg, batch, feat_c, feat_f, frame, t, offs, model, args = _mv_scene("mv_small")
  m, b, fc, _ = _mv_device(model, batch, feat_c, feat_f)
  fine = [getattr(m, k) for k in _FINE]
  g = torch.Generator().manual_seed(4)
  S = cfg["N_samples"] + cfg["N_importance"]
  results = []
  for limit in (rr.TRAIN_ROWS_LIMIT, 7 * S * max(cfg["V_dy"], cfg["V_st"])):  # the second: slices of 7 rays
    monkeypatch.setattr(rr, "TRAIN_ROWS_LIMIT", limit)
    for mod in fine:
      mod.zero_grad(set_to_none=True)
    m.trajectory_basis_fine.grad = None
    ff = tuple(f.to(DEV).requires_grad_(True) if f is not None else None for f in feat_f)
    got = rr.render_rays_mv(frame, t, offs, b, m, Projector(DEV), fc, ff, cfg["N_samples"], args,
                            inv_uniform=cfg["inv_uniform"], N_importance=cfg["N_importance"], det=True,
                            precision="fp32")
    if not results:
      gens = {(o, k): torch.randn(got[o][k].shape, generator=g).to(DEV) for o, ks in _FINE_KEYS.items() for k in ks}
    sum((got[o][k] * v).sum() for (o, k), v in gens.items()).backward()
    grads = [p.grad.clone() for mod in fine for k, p in mod.named_parameters() if k != "s"]
    results.append((got, grads + [m.trajectory_basis_fine.grad.clone(), ff[0].grad.clone(), ff[2].grad.clone()]))
  (a, ga), (bb, gb) = results
  for o in ("outputs_coarse_ref", "outputs_fine_ref", "outputs_fine_ref_dy"):
    for k, v in a[o].items():
      if v.dtype == torch.bool:
        assert torch.equal(bb[o][k], v), (o, k)
      else:
        torch.testing.assert_close(bb[o][k], v, rtol=1e-5, atol=1e-6, msg=lambda s: "%s/%s: %s" % (o, k, s))
  for x, y in zip(gb, ga):
    assert (x - y).norm().item() <= 2e-3 * y.norm().item() + 1e-6
