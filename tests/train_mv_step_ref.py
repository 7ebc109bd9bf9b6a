"""Float64 reference of one fine-stage training step of render_rays_mv (DynibarFF): the differentiable fine pass, a
stand-in loss, backward.

The step is the oracle's `render_rays_mv` (oracle/dynibar_oracle.py, the reference's render_ray.py:600-867) evaluated
in float64 with the library's staged training nets and MotionMLP swapped in for net_fine_dy / net_fine_st /
motion_mlp_fine (train_step_ref._nets: mode "kernel" rounds the operands of exactly the products precision "bf16"
puts on the tensor cores, mode "exact" rounds nothing, precision "fp32").

The coarse pass and the importance resampling are not the subject: the library runs them under no_grad with the
forward path's kernels (tests/test_train_mv_gpu.py checks them bit for bit against the forward call; the forward
stages have float64 tests of their own).  So the reference takes the library's fine depths: `reference(..., z_fine=)`
makes the oracle's `resample_depths` return them for the chunk's rays, and the fine pass is compared at identical
points.  The oracle's coarse pass still runs (under no_grad, as in the reference) and its outputs are returned for an
information-only comparison: it uses the fused bf16 forward kernels, which mode "kernel" does not model.

The loss.  DynibarFF has no criterion (the reference ships no training script for it), so a smooth stand-in is used,
evaluated by torch on both sides (`stand_in_loss`): squared error against seeded targets for the fine rgb, the
fine_dy rgb, depth, the masked render_flows and exp_sf; a seeded linear term on every other differentiable fine output,
so that each reaches the gradients through its own path.  Squared error, not L1, so that no |x| kink sits at exp_sf = 0
in the fresh case.  Every term is a sum over rays divided by the whole batch's R: the loss splits exactly over ray
chunks, so the rays are evaluated in chunks (forward + backward each, gradients accumulating), all of near-equal size
so that every chunk sees the whole batch's tensor-core dispatch (train_step_ref._check_chunk).

`plant` names a deliberate wiring error of the fine pass's glue (PLANTS), made by wrapping oracle functions; nothing
in the oracle or the library is planted.
"""

import contextlib
import copy
from types import SimpleNamespace

import torch

import train_step_ref as TS
from oracle import dynibar_oracle as O

# Planted wiring errors of the fine pass, each scored on PLANT_CASE (tests/test_train_mv_step_gpu.py): it must move some
# compared tensor by at least PLANT_MARGIN times its bf16 bar.
PLANTS = (
    "exp_sf_rows_1",           # exp_sf from the basis rows f +- 1 instead of f +- 2
    "exp_sf_min",              # exp_sf = torch.min of the two expected flows instead of torch.max
    "fine_rows_coarse_basis",  # the fine displacement rows (and exp_sf's) built from trajectory_basis
    "keep_coarse_S",           # the zeroed tail is round(0.1 N_samples) instead of round(0.1 (N_samples + N_importance))
    "static_feat_dy_map",      # the static gather reads fine_featmaps[0] (static view v: dynamic map v mod V_dy)
    "flows_from_undisplaced",  # render_flows from the undisplaced fine points instead of the displaced seq
    "fine_time_zero",          # the fine MotionMLP's time column is 0
)
PLANT_CASE = "edges"  # non-zero motion, a perturbed fine basis, every view count edge
PLANT_MARGIN = 3.0

# Cases.  nvidia: the Nvidia configs' step as tools/train_mv_bench.py runs it, 1024 rays.  linear: linear-depth
# resampling, deterministic u, anti_alias_pooling 0, mask_rgb 1, a ray count that is no multiple of 64 or 128.  fresh:
# coeff_linear zero (weight and bias, as mlp_network.py:602-603 initialises it) and the basis at its DCT init: motion
# is exactly 0, so exp_sf ties on every ray.  edges: 48x64 frames, reference frame 1 (rows f - 2 and f - 3 wrap to the
# last frames), a wide static rig and extra rays off the target frustum (train_step_ref._EDGE_U).  short: 3 + 2
# samples, fine S = 5 (round(0.5) = 0: every sample's coefficients are zeroed).  sliced: nvidia rendered by the
# library in 3 uneven slices (render_ray.TRAIN_ROWS_LIMIT).
_NVIDIA = dict(H=288, W=512, V_dy=7, V_st=11, rays=1024, Sc=64, Si=64, inv=1, aa=1, mrgb=0, det=False, frame_idx=10,
               coeff_std=0.05, basis_jitter=0.05, seed=41, chunk=128, edge_rays=False, slice_rays=None)
CASES = {
    "nvidia": _NVIDIA,
    "linear": dict(_NVIDIA, rays=1031, inv=0, aa=0, mrgb=1, det=True, seed=42),
    "fresh": dict(_NVIDIA, rays=256, coeff_std=0.0, basis_jitter=0.0, seed=43),
    "edges": dict(_NVIDIA, H=48, W=64, rays=96, frame_idx=1, edge_rays=True, seed=44, chunk=None),
    "short": dict(_NVIDIA, H=48, W=64, rays=64, Sc=3, Si=2, seed=45, chunk=None),
    "sliced": dict(_NVIDIA, slice_rays=400),  # slices of 400, 400 and 224 rays
}

OUT_KEYS = {
    "outputs_fine_ref": ("rgb", "rgb_static", "rgb_dy", "depth", "weights", "weights_dy", "weights_st", "alpha",
                         "alpha_dy", "render_flows", "exp_sf", "mask"),
    "outputs_fine_ref_dy": ("rgb", "depth", "weights", "mask"),
}
_SHORT = {"outputs_fine_ref": "fine", "outputs_fine_ref_dy": "fine_dy"}
COARSE_KEYS = ("rgb", "depth", "weights", "mask")
NETS = ("net_fine_dy", "net_fine_st", "motion_mlp_fine")
_COARSE_NETS = ("net_coarse_dy", "net_coarse_st", "motion_mlp")
# the stand-in loss: squared-error terms (output, key, weight) and linear terms (output, key).  exp_sf's weight and
# target scale give its path about half of coeff_linear's gradient on edges and, at zero motion (fresh), where the
# flows' path through the displaced points dominates, about 0.1 %: enough for a wrong tie rule to show
_SQ = (("outputs_fine_ref", "rgb", 1.0), ("outputs_fine_ref_dy", "rgb", 1.0), ("outputs_fine_ref", "depth", 1e-2),
       ("outputs_fine_ref", "render_flows", 1e-2), ("outputs_fine_ref", "exp_sf", 10.0))
_LIN = (("outputs_fine_ref", "rgb_static"), ("outputs_fine_ref", "rgb_dy"), ("outputs_fine_ref", "weights"),
        ("outputs_fine_ref", "weights_dy"), ("outputs_fine_ref", "weights_st"), ("outputs_fine_ref", "alpha"),
        ("outputs_fine_ref", "alpha_dy"), ("outputs_fine_ref_dy", "depth"), ("outputs_fine_ref_dy", "weights"))


def make_case(name, rays=None):
  """Seeded scene, model (CPU, fp32), random draws and loss targets of case `name`; `rays` overrides the ray count."""
  from dynibar_b200 import synthetic
  c = dict(CASES[name], name=name)
  if rays is not None:
    c["rays"] = rays
  batch, feat_c, feat_f, frame, t, offs = synthetic.make_scene(
      H=c["H"], W=c["W"], V_dy=c["V_dy"], V_st=c["V_st"], seed=c["seed"], rays=c["rays"], frame_idx=c["frame_idx"])
  if c["edge_rays"]:
    TS.add_edge_rays(batch, c["H"])
  args = synthetic.make_args(c["aa"], c["mrgb"])
  model, args = synthetic.make_model(c["Sc"], c["Si"], args=args, seed=c["seed"])
  g = torch.Generator().manual_seed(c["seed"] + 1000)
  with torch.no_grad():
    if c["coeff_std"] > 0:  # motion well above zero, so that its gradients are well above rounding
      w = model.motion_mlp_fine.coeff_linear.weight
      w.copy_(torch.randn(w.shape, generator=g) * c["coeff_std"])
    else:
      for mod in (model.motion_mlp, model.motion_mlp_fine):
        mod.coeff_linear.weight.zero_()
        mod.coeff_linear.bias.zero_()
    if c["basis_jitter"] > 0:  # fine rows built from the coarse basis would otherwise give the same values
      b = model.trajectory_basis_fine
      model.trajectory_basis_fine = b + c["basis_jitter"] * torch.randn(b.shape, generator=g)
  R, S, V = batch["ray_o"].shape[0], c["Sc"] + c["Si"], c["V_dy"]
  tgt = {"outputs_fine_ref/rgb": torch.rand(R, 3, generator=g),
         "outputs_fine_ref_dy/rgb": torch.rand(R, 3, generator=g),
         "outputs_fine_ref/depth": torch.rand(R, generator=g) * 8.0 + 1.0,
         "outputs_fine_ref/render_flows": torch.randn(V, R, 2, generator=g) * 3.0,
         "flow_mask": (torch.rand(V, R, 1, generator=g) > 0.3).float(),
         "outputs_fine_ref/exp_sf": torch.randn(R, 3, generator=g) * 0.1}
  shapes = {"rgb_static": (R, 3), "rgb_dy": (R, 3), "depth": (R,)}
  for o, k in _LIN:
    tgt["lin.%s/%s" % (o, k)] = torch.randn(shapes.get(k, (R, S)), generator=g)
  c.update(batch=batch, feat_c=feat_c, feat_f=feat_f, frame=frame, t=t, offs=offs, model=model, args=args, tgt=tgt,
           jitter=torch.rand(R, c["Sc"], generator=g), u=torch.rand(R, c["Si"], generator=g), S=S, R=R)
  return c


def stand_in_loss(ret, tgt, R):
  """The stand-in criterion of a (chunk of a) step: every term a sum over the rays of `ret` divided by the whole batch's
  R.  `tgt` holds the targets of the same rays."""
  loss = 0.0
  for o, k, wt in _SQ:
    e = (ret[o][k] - tgt["%s/%s" % (o, k)]) ** 2
    if k == "render_flows":
      e = e * tgt["flow_mask"]
    loss = loss + wt * e.sum() / R
  for o, k in _LIN:
    loss = loss + (ret[o][k] * tgt["lin.%s/%s" % (o, k)]).sum() / R
  return loss


_TGT_AXIS1 = ("outputs_fine_ref/render_flows", "flow_mask")  # [V_dy, R, ...]; every other target is [R, ...]


def _tgt_rows(tgt, lo, hi):
  return {k: v[:, lo:hi] if k in _TGT_AXIS1 else v[lo:hi] for k, v in tgt.items()}


def spans(R, chunk):
  """Near-equal ray chunks of at least `chunk` rays each (one chunk when chunk is None or R < 2 chunk)."""
  n = 1 if chunk is None else max(1, R // chunk)
  edges = [R * i // n for i in range(n + 1)]
  return list(zip(edges[:-1], edges[1:]))


# ---------------------------------------------------------------------------------------------------------------
# The evaluation
# ---------------------------------------------------------------------------------------------------------------
def _plant_wrappers(plant, S_fine, N_samples, basis_coarse):
  """{oracle name: replacement} that plants `plant` in the fine pass.  The fine pass is the one whose points have
  S_fine = N_samples + N_importance samples (N_importance > 0, so the coarse pass has fewer)."""
  pass0, mc0, esf0, flow0 = O._pass, O.motion_coefficients, O.expected_scene_flow, O.optical_flow
  if plant == "exp_sf_rows_1":
    return {"expected_scene_flow": lambda weights, traj, k: esf0(weights, traj, 1)}
  if plant == "exp_sf_min":
    def expected_scene_flow(weights, traj, k):
      p = (weights[..., None] * (traj[k] - traj[0])).sum(-2)
      m = (weights[..., None] * (traj[-k] - traj[0])).sum(-2)
      return torch.min(p, m)
    return {"expected_scene_flow": expected_scene_flow}
  if plant in ("keep_coarse_S", "fine_time_zero"):
    def motion_coefficients(w, pts, t):
      R, S = pts.shape[:2]
      if S != S_fine:
        return mc0(w, pts, t)
      if plant == "fine_time_zero":
        return mc0(w, pts, t * 0.0)
      xyzt = torch.cat([pts, t.to(pts).reshape(1, 1, 1).expand(R, S, 1)], -1)
      n = int(round(0.1 * N_samples))
      n = n if n > 0 else S
      keep = torch.ones(1, S, 1, dtype=pts.dtype, device=pts.device)
      keep[:, S - n:] = 0.0
      return O.motion_mlp(w, xyzt) * keep
    return {"motion_coefficients": motion_coefficients}

  def _pass(ray_batch, feat_dy, feat_st, pts, z, s, t, frame_idx, offsets, num_vv, w_dy, w_st, w_mo, basis, *a, **k):
    fine = pts.shape[1] == S_fine
    if fine and plant == "fine_rows_coarse_basis":
      basis = basis_coarse
    if fine and plant == "static_feat_dy_map":
      V_st, V_dy = feat_st.shape[0], feat_dy.shape[0]
      feat_st = feat_dy[torch.arange(V_st, device=feat_dy.device) % V_dy]
    out, out_dy, out_st, aux = pass0(ray_batch, feat_dy, feat_st, pts, z, s, t, frame_idx, offsets, num_vv, w_dy,
                                     w_st, w_mo, basis, *a, **k)
    if fine and plant == "flows_from_undisplaced":
      n = out["render_flows"].shape[0]
      out["render_flows"] = flow0(out["weights"], pts[None].expand(n, *pts.shape), ray_batch["src_cameras"][:, :n],
                                  ray_batch["uv_grid"])
    return out, out_dy, out_st, aux
  return {"_pass": _pass}


@contextlib.contextmanager
def _patched(repl):
  saved = {k: getattr(O, k) for k in repl}
  try:
    for k, v in repl.items():
      setattr(O, k, v)
    yield
  finally:
    for k, v in saved.items():
      setattr(O, k, v)


def reference(c, device, mode, z_fine=None, chunk=None, plant=None, dtype=torch.float64):
  """Loss, fine outputs and gradients of case `c`'s step, evaluated on `device`.

  -> {"terms": {"loss": 0-d}, "out": {"fine/rgb": ...}, "grad": {"net_fine_st.base_fc.0.weight": ...,
  "trajectory_basis_fine": ..., "fine_featmaps[0]": ...}, "coarse": {"rgb": ...}}, all detached.
  z_fine: the fine depths [R, N_samples + N_importance] the fine pass is evaluated at (the library's); None keeps the
  oracle's own resampling.  chunk: rays per chunk (None: one chunk).  mode None keeps the oracle's own networks.
  dtype=torch.float32 evaluates the same arithmetic in float32."""
  assert plant is None or plant in PLANTS, plant
  d = lambda x: x.detach().to(device, dtype, copy=True) if torch.is_tensor(x) and x.is_floating_point() else x
  m = c["model"]
  model = SimpleNamespace()
  for name in _COARSE_NETS + NETS:
    w = TS._W({k: d(v).requires_grad_(name in NETS) for k, v in getattr(m, name).state_dict().items()})
    w.shift = float(getattr(getattr(m, name), "shift", 0.0))
    setattr(model, name, w)
  model.trajectory_basis = d(m.trajectory_basis)
  model.trajectory_basis_fine = d(m.trajectory_basis_fine).requires_grad_(True)
  fc = tuple(d(f) for f in c["feat_c"])
  ff = tuple(None if f is None else d(f).requires_grad_(True) for f in c["feat_f"])
  batch = {k: d(v) for k, v in c["batch"].items()}
  tgt = {k: d(v) for k, v in c["tgt"].items()}
  jitter, u = d(c["jitter"]), d(c["u"])
  t = tuple(None if x is None else d(x.float()) for x in c["t"])  # the library embeds the time from an fp32 value
  zf = None if z_fine is None else d(z_fine)
  R, S = c["R"], c["S"]
  parts = spans(R, chunk)
  if mode == "kernel":
    for lo, hi in parts:
      TS._check_chunk(R, hi - lo, S)
  cur = {}
  repl = dict(TS._nets(mode)) if mode is not None else {}
  if zf is not None:
    repl["resample_depths"] = lambda z, weights, n, inv, u=None: zf[cur["lo"]:cur["hi"]]
  if plant is not None:
    repl.update(_plant_wrappers(plant, S, c["Sc"], model.trajectory_basis))
  outs, coarse, total = [], [], 0.0
  with _patched(repl):
    for lo, hi in parts:
      cur.update(lo=lo, hi=hi)
      rb = dict(batch)
      for k in ("ray_o", "ray_d", "uv_grid"):
        rb[k] = batch[k][lo:hi]
      ret = O.render_rays_mv(c["frame"], t, c["offs"], rb, model, None, fc, ff, c["Sc"], c["args"],
                             inv_uniform=bool(c["inv"]), N_importance=c["Si"], det=c["det"], jitter=jitter[lo:hi],
                             u=u[lo:hi])
      loss = stand_in_loss(ret, _tgt_rows(tgt, lo, hi), R)
      loss.backward()
      total = total + loss.detach()
      outs.append({o: {k: ret[o][k].detach() for k in ks} for o, ks in OUT_KEYS.items()})
      coarse.append({k: ret["outputs_coarse_ref"][k].detach() for k in COARSE_KEYS + ("z_vals",)})
  res = {"terms": {"loss": total}, "out": {}, "grad": {}, "coarse": {}}
  for o, ks in OUT_KEYS.items():
    for k in ks:
      res["out"]["%s/%s" % (_SHORT[o], k)] = torch.cat([p[o][k] for p in outs], 1 if k == "render_flows" else 0)
  for k in COARSE_KEYS + ("z_vals",):
    res["coarse"][k] = torch.cat([p[k] for p in coarse], 0)
  for name in NETS:
    for k, v in getattr(model, name).items():
      res["grad"]["%s.%s" % (name, k)] = v.grad
  res["grad"]["trajectory_basis_fine"] = model.trajectory_basis_fine.grad
  for i in (0, 2):
    res["grad"]["fine_featmaps[%d]" % i] = ff[i].grad
  return res


def library(c, device, prec):
  """The same step through the library: render_rays_mv with the fine stage trainable (the differentiable fine pass,
  render_ray._render_mv_train), `stand_in_loss` in fp32, backward; fine feature maps and trajectory_basis_fine are
  leaves.  Same layout as `reference` plus "z_fine" (the fine depths) and the coarse z_vals; every tensor copied to
  the host.  The sliced case renders with TRAIN_ROWS_LIMIT set to give slices of c["slice_rays"] rays."""
  from dynibar_b200 import render_ray as rr, synthetic
  from dynibar_b200.projection import Projector
  dev = torch.device(device)
  m = synthetic.model_to(copy.deepcopy(c["model"]), dev)
  for name in NETS:
    getattr(m, name).requires_grad_(True)
  m.trajectory_basis_fine = m.trajectory_basis_fine.detach().requires_grad_(True)
  fc = tuple(None if f is None else f.to(dev) for f in c["feat_c"])
  ff = tuple(None if f is None else f.to(dev).requires_grad_(True) for f in c["feat_f"])
  limit = rr.TRAIN_ROWS_LIMIT
  if c["slice_rays"]:
    rr.TRAIN_ROWS_LIMIT = c["slice_rays"] * c["S"] * max(c["V_dy"], c["V_st"])
  try:
    ret = rr.render_rays_mv(c["frame"], c["t"], c["offs"], synthetic.to_device(c["batch"], dev), m, Projector(dev),
                            fc, ff, c["Sc"], c["args"], inv_uniform=bool(c["inv"]), N_importance=c["Si"],
                            det=c["det"], jitter=c["jitter"].to(dev), u=c["u"].to(dev), precision=prec)
  finally:
    rr.TRAIN_ROWS_LIMIT = limit
  loss = stand_in_loss(ret, synthetic.to_device(c["tgt"], dev), c["R"])
  loss.backward()
  h = lambda x: None if x is None else x.detach().cpu()
  res = {"terms": {"loss": h(loss)}, "out": {}, "grad": {}, "coarse": {}}
  for o, ks in OUT_KEYS.items():
    for k in ks:
      res["out"]["%s/%s" % (_SHORT[o], k)] = h(ret[o][k])
  for k in COARSE_KEYS + ("z_vals",):
    res["coarse"][k] = h(ret["outputs_coarse_ref"][k])
  res["z_fine"] = h(ret["outputs_fine_ref"]["z_vals"])
  for name in NETS:
    for k, p in getattr(m, name).named_parameters():
      res["grad"]["%s.%s" % (name, k)] = h(p.grad)
  res["grad"]["trajectory_basis_fine"] = h(m.trajectory_basis_fine.grad)
  for i in (0, 2):
    res["grad"]["fine_featmaps[%d]" % i] = h(ff[i].grad)
  return res


# ---------------------------------------------------------------------------------------------------------------
# Comparison
# ---------------------------------------------------------------------------------------------------------------
def errors(got, ref, V_st):
  """{name: (relative L2 error, max |error| / max |reference|)} over the loss, the fine outputs and the gradients
  (train_step_ref.errors)."""
  return TS.errors(got, ref, V_st)


def zero_violations(got, ref):
  """Tensors (and rows of trajectory_basis_fine's gradient) that are exactly zero in the reference but not in `got`:
  a gradient behind a zero factor, or a basis row the step does not read, must come out exactly zero."""
  g, r = TS.flat(got), TS.flat(ref)
  bad = []
  for name, b in r.items():
    a = g[name]
    if b is None or a is None:
      continue
    b, a = b.detach().cpu(), a.detach().cpu().reshape(b.shape)
    if not b.any() and a.any():
      bad.append(name)
    elif name == "grad.trajectory_basis_fine":
      rows = [i for i in range(b.shape[0]) if not b[i].any() and a[i].any()]
      if rows:
        bad.append("%s rows %s" % (name, rows))
  return bad


def zero_tensors(ref):
  """Names of the reference's tensors that are exactly zero, and the zero rows of the basis gradient."""
  r = TS.flat(ref)
  names = [k for k, v in r.items() if v is not None and not v.any()]
  b = r["grad.trajectory_basis_fine"]
  return names, [i for i in range(b.shape[0]) if not b[i].any()]


def coarse_errors(got, ref):
  """Information only: {key: (relative L2, max-abs ratio)} of the coarse outputs (the fused forward kernels)."""
  out = {}
  for k in COARSE_KEYS:
    a, b = got["coarse"][k].double().cpu(), ref["coarse"][k].double().cpu()
    e = a - b
    out[k] = (float(e.norm() / b.norm()) if b.norm() > 0 else float(e.norm()),
              float(e.abs().max() / b.abs().max()) if b.abs().max() > 0 else float(e.abs().max()))
  return out


def view_counts(c):
  """Valid views per sample of undisplaced points at S uniform depths, [R, S] each: (static, dynamic)."""
  return TS.view_counts(c)
