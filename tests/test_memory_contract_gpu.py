"""The memory contract of every product path (include/dynibar_b200.h, "Conventions"), checked with the harness of
tests/memory_contract.py: exact-size workspaces and CUDA `torch.empty` / `torch.empty_like` buffers, each followed by
a 64 KiB guard band, all filled with one byte pattern, 0x00, 0xFF (NaN) or 0x7F (3.39e38).  Memory that reaches the
library any other way (torch.zeros, torch.full, the library's own cudaMalloc) is not poisoned.

Every scenario runs once per pattern.  Rules:
  - every guard band is intact under every pattern (no write past a declared size);
  - deterministic paths (inference in both precisions, the criterion and its gradients, the scene loaders, scoring,
    splatting): every output is bit-identical across the patterns (no read of memory the call did not write);
  - paths with float atomics (the training backward of the nets, the MotionMLP, the encoder and of whole steps):
    forward outputs and losses are bit-identical, every gradient is finite, and every gradient agrees with the 0x00
    run within 4x the spread of two 0x00 runs of the same scenario (relative L2 of all its gradients taken as one
    vector, at least memory_contract.SPREAD_FLOOR).  The test prints that spread.
Accumulating outputs (`d_params` and the other gradients the wrappers zero) start from the wrappers' own zeros.

Shapes sit at the edges of the sizing formulas: rows not a multiple of 64 / 128 / 256, view counts at the fused
kernels' 8- and 16-slot limits and past them (staged), sample counts up to the SIMT attention (192), a call across an
internal chunk, the tensor-core thresholds of training, ragged encoder tiles, criterion rows not a multiple of 8 and
odd image sizes.
"""

import copy
import io
import types

import numpy as np
import pytest
import torch

import memory_contract as mc
import scenes
from dynibar_b200 import synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def check_deterministic(scenario, what):
  runs = {}
  for pat in mc.PATTERNS:
    with mc.poisoned(pat):
      runs["0x%02X" % pat] = mc.flatten(scenario())
  mc.assert_bit_identical(runs, what)


def check_atomic(scenario, what):
  """scenario() -> (forward outputs, gradients).  The gradients are compared as one vector: a gradient that is a sum
  whose terms cancel (a static blending-head bias, say) changes by 1e-3 of its own norm with the order of its float
  atomics, so two 0x00 runs whose atomics happened to add in the same order would set a bar its next run misses."""
  runs = {}
  for label, pat in (("0x00", 0x00), ("0x00 again", 0x00), ("0xFF", 0xFF), ("0x7F", 0x7F)):
    with mc.poisoned(pat):
      fwd, grad = scenario()
      runs[label] = (mc.flatten(fwd), mc.flatten(grad))
  mc.assert_bit_identical({k: v[0] for k, v in runs.items()}, what + " (forward)")
  base = runs["0x00"][1]
  assert base, what
  spread, _ = mc.global_rel_l2(runs["0x00 again"][1], base)
  bar = 4.0 * max(spread, mc.SPREAD_FLOOR)
  errs = {}
  for label in ("0xFF", "0x7F"):
    g = runs[label][1]
    for k in base:
      assert bool(torch.isfinite(g[k]).all()), "%s: gradient %s is not finite under pattern %s" % (what, k, label)
    errs[label] = mc.global_rel_l2(g, base)
  print("\n%s: gradients' spread over two 0x00 runs %.3e (rel. L2 of all gradients); 0xFF %.3e (most in %s), "
        "0x7F %.3e (most in %s); bar %.3e" % (what, spread, *errs["0xFF"], *errs["0x7F"], bar))
  for label, (e, k) in errs.items():
    assert e <= bar, "%s: the gradients under %s are %.3e (rel. L2) off the 0x00 run, most in %s; spread %.3e" % (
        what, label, e, k, spread)


# ---------------------------------------------------------------------------------------------------------------
# inference: render_rays_mv / render_rays_mono
# ---------------------------------------------------------------------------------------------------------------
_BASE = dict(H=36, W=64, inv_uniform=True, anti_alias_pooling=1, mask_rgb=1, stress=True)
RENDER_CASES = {
    # P = 37 x 5 = 185 point rows, 37 x 5 x 8 view rows: no multiple of 64, 128 or 256
    "mono_p37_s5": dict(_BASE, mono=True, V_dy=8, V_st=4, rays=37, N_samples=5, N_importance=0, num_vv=2, seed=41),
    "mv_v1": dict(_BASE, mono=False, V_dy=1, V_st=1, rays=45, N_samples=16, N_importance=4, num_vv=0, seed=42),
    "mv_v8_v9": dict(_BASE, mono=False, V_dy=8, V_st=9, rays=61, N_samples=16, N_importance=4, num_vv=0, seed=43,
                     mask_rgb=0),
    "mono_v16_s64": dict(_BASE, mono=True, V_dy=16, V_st=16, rays=50, N_samples=64, N_importance=0, num_vv=3,
                         seed=44),
    "mv_v17_v32": dict(_BASE, mono=False, V_dy=17, V_st=32, rays=29, N_samples=16, N_importance=4, num_vv=0,
                       seed=45),
    "mv_s128": dict(_BASE, mono=False, V_dy=7, V_st=11, rays=33, N_samples=64, N_importance=64, num_vv=0, seed=46),
    "mv_s192": dict(_BASE, mono=False, V_dy=10, V_st=10, rays=19, N_samples=64, N_importance=128, num_vv=0,
                    seed=47, stress=False),
    # net_rows_per_chunk at S = 128, V = 16 is 2048 rays: one ray under, at and over one chunk
    "mono_r2047": dict(_BASE, mono=True, V_dy=16, V_st=16, rays=2047, N_samples=128, N_importance=0, num_vv=3,
                       seed=48, stress=False),
    "mono_r2048": dict(_BASE, mono=True, V_dy=16, V_st=16, rays=2048, N_samples=128, N_importance=0, num_vv=3,
                       seed=48, stress=False),
    "mono_r2049": dict(_BASE, mono=True, V_dy=16, V_st=16, rays=2049, N_samples=128, N_importance=0, num_vv=3,
                       seed=48, stress=False),
    # the cross-time branch (is_train=True) with virtual views, under no_grad
    "mono_cross_time": dict(scenes.GOLDEN_CONFIGS["mono_train"], rays=37),
}


def _render(cfg, prec):
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  d = lambda x: synthetic.to_device(x, DEV)

  def run():
    m = synthetic.model_to(copy.deepcopy(model), DEV)
    with torch.no_grad():
      if cfg["mono"]:
        return rr.render_rays_mono(frame, t, offs, d(batch), m, d(feat_c), Projector(DEV), cfg["N_samples"], args,
                                   inv_uniform=cfg["inv_uniform"], det=True, is_train="anchor_offset" in cfg,
                                   num_vv=cfg["num_vv"], precision=prec)
      return rr.render_rays_mv(frame, t, offs, d(batch), m, Projector(DEV), d(feat_c), d(feat_f), cfg["N_samples"],
                               args, inv_uniform=cfg["inv_uniform"], N_importance=cfg["N_importance"], det=True,
                               is_train=False, precision=prec)
  return run


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("case", list(RENDER_CASES))
def test_render_rays(case, prec):
  check_deterministic(_render(RENDER_CASES[case], prec), "%s %s" % (case, prec))


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("kind,S", [("dynamic", 1), ("static", 1), ("dynamic", 20), ("static", 192)])
def test_staged_net_inference(kind, S, prec):
  """The staged nets on their own at the sample counts a render does not reach here (1) and at the SIMT attention's
  192; 23 rays x 9 views."""
  import train_stage_ref as tsr
  from dynibar_b200 import render_ray as rr
  c = tsr.make_forward_case(kind, 23, S, 9, kind == "static", kind == "static", seed=S, device=DEV)

  def run():
    mod = copy.deepcopy(c["mod"]).to(DEV).requires_grad_(False)
    with torch.no_grad(), rr.precision_scope(prec):
      if kind == "dynamic":
        return rr.net_dynamic_forward(mod, c["pts"], c["feat"], c["ray_dir"], c["mask"], c["t"])
      return rr.net_static_forward(mod, c["pts"], c["ref_rays"], c["src_rays"], c["feat"], c["ray_diff"], c["mask"])
  check_deterministic(run, "staged %s S=%d %s" % (kind, S, prec))


# ---------------------------------------------------------------------------------------------------------------
# multi-camera renders
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_render_multi_image_nvi(prec):
  """Three target cameras of 12 x 16 rays in chunks of 100: chunks straddle cameras."""
  from dynibar_b200 import render_ray as rr, sample_ray as sr
  from dynibar_b200.projection import Projector
  from dynibar_b200.render_image import render_multi_image_nvi
  H, W = 12, 16
  cfg = dict(scenes.GOLDEN_CONFIGS["mv_small"], H=H, W=W, V_st=11, rays=None, seed=21, stress=False)
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  data = scenes.sampler_data(batch, H, W, cfg["seed"])
  K_mat = sr.parse_camera(batch["camera"])[2][0]

  def run():
    samplers = []
    for off in ((0.0, 0.0, 0.0), (0.045, 0.012, -0.02), (-0.03, -0.017, 0.035)):
      c2w = torch.eye(4)
      c2w[:3, 3] = torch.tensor(off)
      samplers.append(sr.RaySamplerSingleImage(dict(data, camera=synthetic.camera_vector(H, W, K_mat, c2w)[None]),
                                               DEV))
    rays, _, _ = sr.stack_ray_batches([s.get_all() for s in samplers])
    m = synthetic.model_to(copy.deepcopy(model), DEV)
    d = lambda x: synthetic.to_device(x, DEV)
    with torch.no_grad(), rr.precision_scope(prec):
      return render_multi_image_nvi(frame, t, offs, samplers, rays, m, Projector(DEV), 100, cfg["N_samples"], args,
                                    inv_uniform=True, N_importance=cfg["N_importance"], det=True,
                                    coarse_featmaps=d(feat_c), fine_featmaps=d(feat_f), is_train=False)
  check_deterministic(run, "render_multi_image_nvi %s" % prec)


# ---------------------------------------------------------------------------------------------------------------
# training
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("kind,case", [(k, c) for c in ("all_simt", "fwd_tc_only", "ragged", "per_ray_tc")
                                       for k in ("dynamic", "static")])
def test_net_training(kind, case, prec):
  """The staged nets' training forward and backward on both sides of the 128-row forward and the 2048-row backward
  tensor-core thresholds (train_stage_ref.dispatch)."""
  import train_stage_ref as tsr
  from test_train_stage_gpu import _library
  R, S, V, aa, mrgb = tsr.NET_CASES[case]
  c = tsr.make_net_case(kind, R, S, V, aa, mrgb, seed=R + V)

  def run():
    got = _library(c, prec)
    return {"out": got.pop("out")}, got
  check_atomic(run, "%s %s %s" % (kind, case, prec))


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("case", ["n2047", "n2048", "n2049"])
def test_motion_training(case, prec):
  import train_stage_ref as tsr
  from test_train_stage_gpu import _library
  N, nb = tsr.MOTION_CASES[case]
  c = tsr.make_motion_case(N, nb, seed=N + nb)

  def run():
    got = _library(c, prec)
    return {"out": got.pop("out")}, got
  check_atomic(run, "motion %s %s" % (case, prec))


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("case", ["below_2048", "at_2048", "ragged"])
def test_encoder_training(case, prec):
  import encoder_ref as er
  from test_encoder_train_gpu import _library
  c = er.make_case(case)

  def run():
    got = _library(c, prec)
    return {k: got.pop(k) for k in ("coarse", "fine")}, got
  check_atomic(run, "encoder %s %s" % (case, prec))


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("slice_rays", [None, 64])
def test_mono_step_backward(slice_rays, prec):
  """train_step.mono_step_backward on the edge-ray case, in one call and in 64-ray slices (105 rays)."""
  import train_step_ref as T
  from test_train_sliced_gpu import step
  c = T.make_case("edges_occ1")
  R = c["batch"]["ray_o"].shape[0]

  def run():
    res = step(c, prec, slice_rays or R)
    return res["terms"], res["grad"]
  check_atomic(run, "mono_step_backward %s slices of %s" % (prec, slice_rays or R))


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_render_rays_mv_fine_stage_step(prec):
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  from test_train_mv_gpu import _FINE, _mv_device, _mv_scene
  cfg, batch, feat_c, feat_f, frame, t, offs, model, args = _mv_scene("mv_nvidia", 37)
  g = torch.Generator().manual_seed(7)

  def run():
    m, b, fc, ff = _mv_device(copy.deepcopy(model), batch, feat_c, feat_f)
    got = rr.render_rays_mv(frame, t, offs, b, m, Projector(DEV), fc, ff, cfg["N_samples"], args, precision=prec,
                            inv_uniform=cfg["inv_uniform"], N_importance=cfg["N_importance"], det=True,
                            is_train=True)
    out = got["outputs_fine_ref"]
    g.manual_seed(7)
    sum((v * torch.randn(v.shape, generator=g).to(DEV)).sum() for k, v in sorted(out.items())
        if torch.is_tensor(v) and v.requires_grad).backward()
    grads = {"%s.%s" % (n, k): p.grad for n in _FINE for k, p in getattr(m, n).named_parameters()}
    grads["trajectory_basis_fine"] = m.trajectory_basis_fine.grad
    grads.update({"feat_f[%d]" % i: f.grad for i, f in enumerate(ff) if f is not None})
    return got, grads
  check_atomic(run, "render_rays_mv fine stage %s" % prec)


# ---------------------------------------------------------------------------------------------------------------
# the criterion (no float atomics: gradients too must be bit-identical)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1003, 5])
def test_mono_step_loss(R):
  import test_loss_gpu as TL
  from dynibar_b200 import criterion as cr
  ret, rb = TL.generated(R, 64, 3, 900 + R)

  def run():
    leaves = {o: {k: v.to(DEV).requires_grad_(k in TL.GRAD_KEYS.get(o, ())) if v.is_floating_point()
                  else v.to(DEV) for k, v in d.items()} for o, d in ret.items()}
    rbd = {k: v.to(DEV) for k, v in rb.items()}
    table = cr.mono_step_table(leaves, rbd, TL.loss_args(), 0)
    table[0].backward()
    return table, {o: {k: v.grad for k, v in d.items() if torch.is_tensor(v) and v.grad is not None}
                   for o, d in leaves.items()}
  check_deterministic(run, "mono_step_loss R=%d" % R)


def test_criterion_slices():
  """slice_rows into one batch buffer (R = 1003 = 504 + 499 rays, not a multiple of 8), batch_table, slice_loss."""
  import test_loss_gpu as TL
  from dynibar_b200 import autograd as ag, criterion as cr
  from test_train_sliced_gpu import _cut
  R = 1003
  ret, rb = TL.generated(R, 64, 3, 77)
  args = TL.loss_args()

  def run():
    partial = torch.empty(int(ag.lib.dyn_mono_loss_workspace_bytes(R)), dtype=torch.uint8, device=DEV)
    parts = []
    for lo, hi in ((0, 504), (504, R)):
      p = {o: {k: v.to(DEV).requires_grad_(k in TL.GRAD_KEYS.get(o, ())) if v.is_floating_point() else v.to(DEV)
               for k, v in _cut(d, lo, hi).items()} for o, d in ret.items()}
      r = {k: v.to(DEV) for k, v in _cut(rb, lo, hi).items()}
      wt, dims = cr.slice_rows(p, r, args, 0, partial, lo)
      parts.append((p, r))
    table = cr.batch_table(partial, wt, R, dims)
    for p, r in parts:
      cr.slice_loss(p, r, args, 0, table).backward()
    return table, [{o: {k: v.grad for k, v in d.items() if torch.is_tensor(v) and v.grad is not None}
                    for o, d in p.items()} for p, _ in parts]
  check_deterministic(run, "criterion slices")


# ---------------------------------------------------------------------------------------------------------------
# scenes, scoring, splatting
# ---------------------------------------------------------------------------------------------------------------
def test_monocular_scene_batches(tmp_path):
  import mono_scene_ref as msr
  import test_mono_scene_gpu as TM
  from dynibar_b200 import mono_scene, sample_ray
  golden = msr.load_golden(TM.GOLDEN)
  c = golden["cases"][0]
  raw = dict(np.load(io.BytesIO(golden["scenes"][c["scene"]]["raw"])))
  path = msr.write_scene(str(tmp_path / "dense"), raw)

  def run():
    s = mono_scene.MonocularScene(path, TM._args(golden, c), torch.device(DEV))
    s.set_epoch(c["epoch"])
    out = []
    for k in range(2):
      sample_ray.rng = np.random.RandomState(c["pixel_seed"] + k)
      td, rb = s.sample(np.random.RandomState(c["seed"] + k), golden["n_rand"], c["sample_mode"])
      out.append(({k: v for k, v in td.items() if torch.is_tensor(v)}, rb))
    return out
  check_deterministic(run, "MonocularScene.sample")


def test_nvidia_scene_time_step(tmp_path):
  import nvi_scene_ref as nsr
  import test_nvi_scene_gpu as TN
  from dynibar_b200 import nvidia_scene as ns
  golden = nsr.load_golden(TN.GOLDEN)
  name, s = next(iter(golden["scenes"].items()))
  path = nsr.write_files(str(tmp_path / name / "dense"), s["files"])
  img_i = sorted({int(it["img_i"]) for it in s["items"]})[0]

  def run():
    scene = ns.NvidiaScene(path, types.SimpleNamespace(mask_static=bool(s["mask_static"])), DEV)
    return scene.time_step(img_i)
  check_deterministic(run, "NvidiaScene.time_step")


def test_bullet_time_group_batch_and_frames(tmp_path):
  import bt_scene_ref as bsr
  import test_bt_scene_gpu as TB
  from dynibar_b200 import bt_scene
  from dynibar_b200.projection import Projector
  golden = bsr.load_golden(TB.GOLDEN)
  case = golden["cases"][0]
  root = bsr.write_scene(str(tmp_path / case["scene"] / "dense"), golden["scenes"][case["scene"]])
  args = TB._args(case)

  def run():
    scene = bt_scene.BulletTimeScene(root, args, DEV)
    model = TB._model()
    return [scene.group_batch(g) for g in range(min(2, len(scene)))], list(scene.sweep(model, Projector(DEV), args))
  check_deterministic(run, "BulletTimeScene group_batch / sweep")


@pytest.mark.parametrize("H,W", [(45, 71), (37, 8)])
def test_image_scores_odd_sizes(H, W):
  import metrics_ref as mr
  from dynibar_b200 import metrics
  pred, gt, dyn = mr.eval_case(3, H, W, seed=H + W)

  def run():
    return [metrics.score_views(torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV),
                                torch.from_numpy(dyn).to(DEV)),
            metrics.score_views(torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV))]
  check_deterministic(run, "score_views %dx%d" % (H, W))


@pytest.mark.parametrize("case", ["odd", "edges", "batch"])
def test_splatting_odd_sizes(case):
  import virtual_views_ref as vr
  from dynibar_b200 import virtual_views as vv
  frame, flow, metric = vr.splat_case(case)

  def run():
    return vv.splatting_function("softmax", frame.to(DEV), flow.to(DEV), metric.to(DEV))
  check_deterministic(run, "splatting %s" % case)


def test_forward_splat_and_virtual_views():
  import virtual_views_ref as vr
  from dynibar_b200 import virtual_views as vv
  imgs, d, r, t, k = vr.forward_case("const")
  img, disp, K, ref2w, tgt = vr.frame_case()

  def run():
    return (vv.render_forward_splat(imgs.to(DEV), d.to(DEV), r, t, k, k),
            vv.sobel_fg_alpha(d[:, None].to(DEV), "sobel", beta=10.0),
            vv.render_virtual_views(torch.from_numpy(img).to(DEV), torch.from_numpy(disp).to(DEV), K, ref2w, tgt))
  check_deterministic(run, "forward splat / virtual views")
