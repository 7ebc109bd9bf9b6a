"""Float64 reference of one monocular training step: render_rays_mono(is_train=True), the criterion, backward.

The step is the oracle's `render_rays_mono` (oracle/dynibar_oracle.py, the reference's render_ray.py:870-1277 with its
cross-time branch) evaluated in float64 with two kinds of parts swapped in:
  * the networks: oracle.net_dynamic / net_static / motion_mlp are replaced, for the duration of the evaluation, by
    train_stage_ref's restatements of the library's staged training nets and MotionMLP.  Mode "kernel" rounds the
    operands of exactly the products the library's precision "bf16" puts on the tensor cores (train_stage_ref.dispatch),
    mode "exact" rounds nothing (precision "fp32");
  * the loss: loss_ref.mono_step_loss (train.py:300-456).
Everything else (sampling, displacement, projection and bilinear gathers, compositing, optical flow, the
cross-time branch) is the oracle's own code, in float64.

`reference` returns the nine loss terms, the outputs the criterion reads, and the gradient of the loss with respect to
every parameter of net_coarse_dy / net_coarse_st / motion_mlp, trajectory_basis and featmaps[0..2].  It evaluates
the rays in chunks to keep device memory modest: the nets are per ray, and the criterion couples rays only through
normalisers and counts built from supervision, masks or detached forward values (loss_ref.step_denominators).  Those
come from a no-grad pass over all chunks; then each chunk runs forward + backward with them held fixed and the
gradients accumulate.  A chunk must see the same tensor-core dispatch as the whole batch (`_check_chunk`).

`plant` names a deliberate wiring error of the step's glue (PLANTS), used to show that the bars of
tests/test_train_step_gpu.py would catch it.  Plants are made by wrapping the oracle's `_pass` / `_cross_time` or by
rerouting a feature map's gradient; nothing in the oracle or the library is planted.
"""

import contextlib
import copy
from types import SimpleNamespace

import torch

import loss_ref
import train_stage_ref as tsr
from oracle import dynibar_oracle as O

# Planted wiring errors (scored on the edges case in tests/test_train_step_gpu.py; each must move at least one
# compared quantity by PLANT_MARGIN times its bar).  None of the suggested plants is invisible.  "render_flows over
# all dynamic views instead of 6" cannot be compared at all (the supervision has 6 flow views, so the loss does not
# broadcast); its near relative, the flow views taken one slot late, is planted instead.
PLANTS = (
    "anchor_raw_st_detached",  # the anchor composite reads a detached raw_st: no anchor gradient reaches net_static
    "anchor_feat_to_f0",       # the anchor gather's feature gradient lands in featmaps[0] instead of featmaps[1]
    "sf_seq_shifted",          # sf_seq built from offsets -3..2 instead of -2..3 (traj[o-1] - traj[o-2])
    "occ_not_detached",        # occ_weights / occ_weight_map keep their graph (the reference detaches them)
    "flow_views_shifted",      # render_flows from the dynamic views 1..6 instead of 0..5
    "anchor_basis_detached",   # the basis rows of the anchor's offsets (traj_a0 and seq_a) detached
    "vv_rows_displaced",       # the virtual-view rows of seq displaced by the +1 trajectory instead of staying put
)
PLANT_MARGIN = 3.0

# the shipped config's loss weights (configs/train_kid-running.txt of the reference)
LOSS_ARGS = dict(w_disp=1e-1, w_flow=1e-2, w_cycle=0.1, cycle_factor=0.1, anneal_cycle=True, w_reg=0.05,
                 w_skew_entropy=5e-4, w_distortion=1e-3, decay_rate=10.0, init_decay_epoch=400)

# Cases.  shipped: the step DESIGN §3.7 runs with the shipped config's views -- 1024 rays x 64 samples (N_rand 3072
# does not fit the saved activations in 80 GB), 288x512 frames, 7 source + 3 virtual dynamic views, 14 static views,
# the anchor stack two frames away, anti_alias_pooling 0, mask_rgb 1, occ_weights_mode 0.  late: the same step at an
# epoch past 5 init_decay_epoch (static_dy on, dynamic_rgb off).  edges: about 100 rays on 48x64 frames with the
# reference frame at 1 (basis rows wrap, anchor cycle lists shrink), the anchor one frame away, anti-aliasing on,
# occ_weights_mode 1 / 2, a wide static rig and extra rays off the target frustum (no valid static view; samples with
# fewer than 2 valid dynamic views).
_SHIPPED = dict(H=288, W=512, V_dy=10, V_st=14, num_vv=3, rays=1024, S=64, aa=0, mrgb=1, occ=0, frame_idx=10,
                anchor_offset=2, epoch=0, seed=21, chunk=128, edge_rays=False)
_EDGES = dict(H=48, W=64, V_dy=10, V_st=14, num_vv=3, rays=96, S=64, aa=1, mrgb=1, occ=1, frame_idx=1,
              anchor_offset=1, epoch=0, seed=23, chunk=None, edge_rays=True)
CASES = {
    "shipped": _SHIPPED,
    "late": dict(_SHIPPED, epoch=5 * LOSS_ARGS["init_decay_epoch"] + 7, seed=22),
    "edges_occ1": _EDGES,
    "edges_occ2": dict(_EDGES, occ=2, anchor_offset=-1, seed=24),
}
# pixel columns of the extra rays of the edges cases: just outside the frame (some views see their samples) to far
# outside (none does)
_EDGE_U = (-1.5, -4.0, -9.0, -20.0, -45.0, -400.0, 66.0, 75.0, 500.0)

OUT_KEYS = {
    "outputs_coarse_ref": ("rgb", "rgb_dy", "rgb_static", "depth", "weights", "weights_dy", "weights_st",
                           "render_flows", "s_vals", "mask"),
    "outputs_coarse_ref_dy": ("rgb", "mask"),
    "outputs_coarse_anchor": ("rgb", "mask", "occ_weights", "occ_weight_map", "pts_traj_ref", "pts_traj_anchor",
                              "sf_seq"),
    "outputs_coarse_anchor_dy": ("rgb", "mask", "occ_weight_map"),
}
_SHORT = {"outputs_coarse_ref": "ref", "outputs_coarse_ref_dy": "ref_dy", "outputs_coarse_anchor": "anchor",
          "outputs_coarse_anchor_dy": "anchor_dy"}
_RAY_AXIS1 = ("render_flows", "pts_traj_ref", "pts_traj_anchor", "sf_seq")  # [n, R, ...]; the rest [R, ...]
NETS = ("net_coarse_dy", "net_coarse_st", "motion_mlp")


def make_case(name):
  """Seeded scene, model (CPU, fp32), supervision, jitter and loss arguments of case `name`."""
  from dynibar_b200 import synthetic
  c = dict(CASES[name], name=name)
  batch, feat, _, frame, t, offs = synthetic.make_scene(
      H=c["H"], W=c["W"], V_dy=c["V_dy"], V_st=c["V_st"], num_vv=c["num_vv"], seed=c["seed"], rays=c["rays"],
      frame_idx=c["frame_idx"], anchor_offset=c["anchor_offset"])
  if c["edge_rays"]:
    add_edge_rays(batch, c["H"])
  args = synthetic.make_args(c["aa"], c["mrgb"], c["occ"])
  model, args = synthetic.make_model(c["S"], 0, args=args, seed=c["seed"], mono=True)
  args = SimpleNamespace(**dict(vars(args), **LOSS_ARGS))
  with torch.no_grad():  # motion well above the zero initialisation, so that its gradients are well above rounding
    model.motion_mlp.coeff_linear.weight.normal_(0.0, 0.05)
  R = batch["ray_o"].shape[0]
  g = torch.Generator().manual_seed(c["seed"] + 1000)
  motion = (torch.rand(R, generator=g) > 0.5).float()
  sup = {"rgb": torch.rand(R, 3, generator=g), "disp": torch.rand(R, generator=g) * 0.5 + 0.05,
         "motion_mask": motion, "static_mask": 1.0 - motion,
         "flows": torch.randn(6, R, 2, generator=g) * 3.0,
         "masks": (torch.rand(6, R, 1, generator=g) > 0.3).float()}
  c.update(batch=batch, featmaps=feat, frame=frame, t=t, offs=offs, model=model, args=args, sup=sup,
           jitter=torch.rand(R, c["S"], generator=g))
  return c


def add_edge_rays(batch, H):
  """Widens the static rig and appends the rays of _EDGE_U to `batch`, in place."""
  batch["static_src_cameras"][0, :, 18 + 3] *= 6.0  # baseline 0.48: pooling weights e_v - min e well above 0
  K = batch["camera"][0, 2:18].reshape(4, 4)[:3, :3]
  uv = torch.tensor([[u, 0.25 * H + 3.0 * i] for i, u in enumerate(_EDGE_U)])
  d = torch.cat([uv, torch.ones(len(_EDGE_U), 1)], 1) @ torch.inverse(K).t()
  batch["ray_o"] = torch.cat([batch["ray_o"], torch.zeros(len(_EDGE_U), 3)])
  batch["ray_d"] = torch.cat([batch["ray_d"], d])
  batch["uv_grid"] = torch.cat([batch["uv_grid"], uv])


def view_counts(c):
  """Valid views per sample of the undisplaced points (no jitter), [R, S] each: (static, dynamic)."""
  b = c["batch"]
  pts, _, _ = O.sample_along_ray(b["ray_o"], b["ray_d"], b["depth_range"], c["S"], True)
  out = []
  for k in ("static_src_rgbs", "src_rgbs"):
    cams = b[k.replace("rgbs", "cameras")]
    V = cams.shape[1]
    feat = torch.zeros(V, 1, c["H"] // 4, c["W"] // 4)
    _, _, m = O.project_gather(pts, pts[None].repeat(V, 1, 1, 1), b["camera"], b[k], cams, feat)
    out.append(m[..., 0].sum(2))
  return tuple(out)


# ---------------------------------------------------------------------------------------------------------------
# The evaluation
# ---------------------------------------------------------------------------------------------------------------
class _W(dict):
  """state_dict of leaf tensors; the oracle reads `shift` off what it is handed as net_coarse_dy."""
  shift = 0.0


def _nets(mode):
  def net_dynamic(w, pts, rgb_feat, ray_dir, mask, t, shift=0.0):
    return tsr.net_dynamic(w, pts, rgb_feat, ray_dir, mask, t, shift, mode)

  def net_static(w, pts, ref_rays, src_rays, rgb_feat, ray_diff, mask, anti_alias_pooling=True, mask_rgb=False):
    return tsr.net_static(w, pts, ref_rays, src_rays, rgb_feat, ray_diff, mask, anti_alias_pooling, mask_rgb, mode)

  def motion_mlp(w, xyzt):  # the library evaluates the MotionMLP over all R S points of a call as rows
    return tsr.motion_mlp(w, xyzt.reshape(-1, 4), mode).reshape(*xyzt.shape[:-1], -1)

  return dict(net_dynamic=net_dynamic, net_static=net_static, motion_mlp=motion_mlp)


def _plant_wrappers(plant):
  """{oracle name: replacement} that plants `plant` in the step's glue."""
  pass0, cross0 = O._pass, O._cross_time
  if plant == "flow_views_shifted":
    def _pass(ray_batch, *a, **k):
      out, out_dy, out_st, aux = pass0(ray_batch, *a, **k)
      out["render_flows"] = O.optical_flow(out["weights"], aux["seq"][1:7], ray_batch["src_cameras"][:, 1:7],
                                           ray_batch["uv_grid"])
      return out, out_dy, out_st, aux
    return {"_pass": _pass}
  if plant == "vv_rows_displaced":
    def _pass(ray_batch, f_dy, f_st, pts, z, s, t, frame_idx, offsets, num_vv, *a, **k):
      return pass0(ray_batch, f_dy, f_st, pts, z, s, t, frame_idx, list(offsets) + [1] * num_vv, 0, *a, **k)
    return {"_pass": _pass}

  def _cross_time(ray_batch, feat_anchor, pts, z, aux, frame_idx, time_embedding, time_offset, num_vv, w_dy, w_mo,
                  basis, shift, occ_mode, out_ref, out_ref_dy):
    if plant == "anchor_raw_st_detached":
      aux = dict(aux, raw_st=aux["raw_st"].detach())
    ret = cross0(ray_batch, feat_anchor, pts, z, aux, frame_idx, time_embedding, time_offset, num_vv, w_dy, w_mo,
                 basis.detach() if plant == "anchor_basis_detached" else basis, shift, occ_mode, out_ref, out_ref_dy)
    a, a_dy = ret["outputs_coarse_anchor"], ret["outputs_coarse_anchor_dy"]
    if plant == "sf_seq_shifted":
      tr = lambda o: O.traj_offset(aux["coeff"], basis[frame_idx[0] + o])
      a["sf_seq"] = torch.stack([tr(o - 1) - tr(o - 2) for o in (-2, -1, 0, 1, 2, 3)], 0)
    if plant == "occ_not_detached":
      ref_idx, anc_idx = frame_idx
      key = {0: "weights_dy" if abs(ref_idx - anc_idx) > 1 else "weights", 1: "weights_dy", 2: "weights"}[occ_mode]
      occ, occ_dy = out_ref[key] - a[key], out_ref_dy["weights"] - a_dy["weights"]
      a["occ_weights"], a["occ_weight_map"] = 1.0 - occ.abs(), 1.0 - occ.sum(1).abs()
      a_dy["occ_weights"], a_dy["occ_weight_map"] = 1.0 - occ_dy.abs(), 1.0 - occ_dy.sum(1).abs()
    return ret
  return {"_cross_time": _cross_time}


@contextlib.contextmanager
def _swapped(mode, plant):
  """The oracle with the library's nets (and `plant`) in place of its own, restored on exit."""
  assert plant is None or plant in PLANTS, plant
  repl = _nets(mode) if mode is not None else {}
  if plant is not None and plant != "anchor_feat_to_f0":
    repl.update(_plant_wrappers(plant))
  saved = {k: getattr(O, k) for k in repl}
  try:
    for k, v in repl.items():
      setattr(O, k, v)
    yield
  finally:
    for k, v in saved.items():
      setattr(O, k, v)


def _check_chunk(R, chunk, S):
  """Every product the library dispatches by row count (train_stage_ref.dispatch: 128 forward, 2048 backward) must
  land on the same side in a chunk as in the whole batch: per-ray rows (ref_feature_fc, rgb_fc.0's direction
  columns) at R, per-point rows at R S, per-(point, view) rows at R S V."""
  for lim in (128, 2048):
    assert (R >= lim) == (chunk >= lim), (R, chunk, lim)
    assert (R * S >= lim) == (chunk * S >= lim), (R, chunk, S, lim)


def _cat(parts):
  return {o: {k: torch.cat([p[o][k] for p in parts], 1 if k in _RAY_AXIS1 else 0) for k in ks}
          for o, ks in OUT_KEYS.items()}


def reference(c, device, mode, chunk=None, plant=None, dtype=torch.float64):
  """Loss terms, criterion inputs and gradients of case `c`'s step, evaluated on `device`.

  -> {"terms": {name: 0-d}, "out": {"ref/rgb": ...}, "grad": {"net_coarse_st.base_fc.0.weight": ...,
  "trajectory_basis": ..., "featmaps[1]": ...}}, all detached.  chunk: rays per chunk (None: one chunk).
  mode None keeps the oracle's own networks (its fp32 restatement, differentiated by torch autograd).
  dtype=torch.float32 evaluates the same arithmetic in float32, an estimate of how far fp32 arithmetic alone drifts
  from the float64 evaluation."""
  d = lambda x: x.detach().to(device, dtype, copy=True) if torch.is_tensor(x) and x.is_floating_point() else x
  m = c["model"]
  model = SimpleNamespace()
  for name in NETS:
    w = _W({k: d(v).requires_grad_(True) for k, v in getattr(m, name).state_dict().items()})
    w.shift = float(getattr(getattr(m, name), "shift", 0.0))
    setattr(model, name, w)
  model.trajectory_basis = d(m.trajectory_basis).requires_grad_(True)
  fm = tuple(d(f).requires_grad_(True) for f in c["featmaps"])
  fm_in = fm
  if plant == "anchor_feat_to_f0":  # featmaps[1]'s values, featmaps[0]'s gradient
    fm_in = (fm[0], fm[1].detach() + (fm[0] - fm[0].detach()), fm[2])
  batch = {k: d(v) for k, v in c["batch"].items()}
  sup = {k: d(v) for k, v in c["sup"].items()}
  jitter = d(c["jitter"])
  t = tuple(d(x.float()) for x in c["t"])  # the library embeds the times from fp32 values
  args, epoch, S = c["args"], c["epoch"], c["S"]
  R = batch["ray_o"].shape[0]
  chunk = R if chunk is None else min(chunk, R)
  if mode == "kernel":
    _check_chunk(R, chunk, S)
  spans = [(lo, min(R, lo + chunk)) for lo in range(0, R, chunk)]

  def render(lo, hi):
    rb = dict(batch)
    for k in ("ray_o", "ray_d", "uv_grid"):
      rb[k] = batch[k][lo:hi]
    return O.render_rays_mono(c["frame"], t, c["offs"], rb, model, fm_in, None, S, args, inv_uniform=True, det=False,
                              is_train=True, num_vv=c["num_vv"], jitter=jitter[lo:hi])

  def sup_of(lo, hi):
    return {k: v[:, lo:hi] if k in ("flows", "masks") else v[lo:hi] for k, v in sup.items()}

  with _swapped(mode, plant):
    if len(spans) == 1:
      ret = render(0, R)
      loss, terms = loss_ref.mono_step_loss(ret, sup, args, epoch)
      loss.backward()
      outs = _cat([ret])
    else:
      with torch.no_grad():
        outs = _cat([render(lo, hi) for lo, hi in spans])
        den = loss_ref.step_denominators(outs, sup, args, epoch)
      terms = None
      for lo, hi in spans:
        loss, tp = loss_ref.mono_step_loss(render(lo, hi), sup_of(lo, hi), args, epoch, den)
        loss.backward()
        terms = tp if terms is None else {k: terms[k] + v for k, v in tp.items()}
  res = {"terms": terms, "out": {}, "grad": {}}
  for o, ks in OUT_KEYS.items():
    for k in ks:
      res["out"]["%s/%s" % (_SHORT[o], k)] = outs[o][k].detach()
  for name in NETS:
    for k, v in getattr(model, name).items():
      res["grad"]["%s.%s" % (name, k)] = v.grad
  res["grad"]["trajectory_basis"] = model.trajectory_basis.grad
  for i, f in enumerate(fm):
    res["grad"]["featmaps[%d]" % i] = f.grad
  return res


def library(c, device, prec):
  """The same step through the library, as train.py runs it: render_rays_mono(is_train=True) over the whole batch,
  criterion.mono_step_loss, backward; feature maps and trajectory_basis are leaves.  Same layout as `reference`,
  every tensor copied to the host."""
  from dynibar_b200 import criterion, render_ray as rr, synthetic
  from dynibar_b200.projection import Projector
  dev = torch.device(device)
  m = synthetic.model_to(copy.deepcopy(c["model"]), dev)
  for name in NETS:
    getattr(m, name).requires_grad_(True)
  m.trajectory_basis = m.trajectory_basis.detach().requires_grad_(True)
  fm = tuple(f.to(dev).requires_grad_(True) for f in c["featmaps"])
  ret = rr.render_rays_mono(c["frame"], c["t"], c["offs"], synthetic.to_device(c["batch"], dev), m, fm, Projector(dev),
                            c["S"], c["args"], inv_uniform=True, det=False, is_train=True, num_vv=c["num_vv"],
                            jitter=c["jitter"].to(dev), precision=prec)
  loss, terms = criterion.mono_step_loss(ret, synthetic.to_device(c["sup"], dev), c["args"], c["epoch"])
  loss.backward()
  h = lambda x: None if x is None else x.detach().cpu()
  res = {"terms": {k: h(v) for k, v in terms.items()}, "out": {}, "grad": {}}
  for o, ks in OUT_KEYS.items():
    for k in ks:
      res["out"]["%s/%s" % (_SHORT[o], k)] = h(ret[o][k])
  for name in NETS:
    for k, p in getattr(m, name).named_parameters():
      res["grad"]["%s.%s" % (name, k)] = h(p.grad)
  res["grad"]["trajectory_basis"] = h(m.trajectory_basis.grad)
  for i, f in enumerate(fm):
    res["grad"]["featmaps[%d]" % i] = h(f.grad)
  return res


# ---------------------------------------------------------------------------------------------------------------
# Comparison
# ---------------------------------------------------------------------------------------------------------------
def _companion(name, V_st):
  """Gradients whose terms cancel are measured against the weight gradient of the same layer
  (train_stage_ref.companion)."""
  net, _, k = name.partition(".")
  kind = {"net_coarse_dy": "dynamic", "net_coarse_st": "static", "net_fine_dy": "dynamic",
          "net_fine_st": "static"}.get(net)
  cn = tsr.companion(kind, k, V_st) if kind else None
  return "%s.%s" % (net, cn) if cn else None


def flat(res):
  """{"term.<name>" / "out.<key>" / "grad.<name>": tensor} of one result; gradients that are None (a parameter the
  loss does not reach) count as zeros of the parameter's shape only when the other side has a tensor."""
  f = {}
  for part in ("terms", "out", "grad"):
    for k, v in res[part].items():
      f["%s.%s" % ({"terms": "term"}.get(part, part), k)] = v
  return f


def errors(got, ref, V_st):
  """{name: (relative L2 error, max |error| / max |reference|)} over every tensor of `ref`."""
  g, r = flat(got), flat(ref)
  out = {}
  for name, b in r.items():
    a = g[name]
    if a is None and b is None:
      continue
    b = torch.zeros(a.shape) if b is None else b.detach().double().cpu()
    a = torch.zeros(b.shape) if a is None else a.detach().double().cpu().reshape(b.shape)
    e = a - b
    cn = _companion(name[len("grad."):], V_st) if name.startswith("grad.") else None
    scale = r["grad." + cn].detach().double().cpu() if cn else b
    nb, mb = float(scale.norm()), float(scale.abs().max()) if scale.numel() else 0.0
    en, em = float(e.norm()), float(e.abs().max()) if e.numel() else 0.0
    out[name] = (en / nb if nb > 0 else en, em / mb if mb > 0 else em)
  return out
