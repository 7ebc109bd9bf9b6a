"""dynibar_b200.criterion on the GPU against the torch restatement of the reference's criterion (tests/loss_ref.py)
evaluated in float64 on the same inputs, and differentiated by torch autograd.

The inputs are the output dicts of a real `render_rays_mono(is_train=True)` call on the training scene of
test_train_gpu.py (so masks, occ_weights and the number K of cycle offsets are what training sees), cut loose from the
renderer as leaves; supervision is seeded (scenes.sampler_data).  Bars: every component rel. 2e-5; gradients rtol 2e-4,
atol 1e-6 * max|g| per tensor.  The last test runs a whole training step."""

import copy
from types import SimpleNamespace

import pytest
import torch

import loss_ref
import scenes
from dynibar_b200 import synthetic

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
