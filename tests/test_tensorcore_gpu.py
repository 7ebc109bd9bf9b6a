"""Tensor-core (wgmma) path: the tensor-core linear layer against a torch reference with
the same operand rounding, and DYN_PREC_BF16 end-to-end parity.

Tolerances (stated, north_star "within a stated floating-point tolerance"):
  * one layer: operands rounded to bf16 exactly like the kernel, fp32
    accumulation -> only summation order differs: rtol 1e-4 / atol 1e-4.
  * end to end in DYN_PREC_BF16 vs the fp32 reference outputs: composited rgb
    |err| <= 2e-3 and PSNR >= 50 dB; depth relative error <= 2e-3; per-sample
    weights |err| <= 2e-3.
"""

import pytest
import torch

import scenes
from dynibar_b200 import synthetic
from oracle import dynibar_oracle as orc
from util import assert_close_frac

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _linear_tc(x, w, b, act):
  from dynibar_b200 import _lib
  M, K = x.shape
  N = w.shape[0]
  y = torch.empty(M, N, device=DEV)
  nbytes = _lib.lib.dyn_linear_tc_packed_bytes(N, K)
  ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
  _lib.check(_lib.lib.dyn_linear_tc(x.data_ptr(), K, w.data_ptr(), b.data_ptr() if b is not None else None,
                                    M, N, K, act, y.data_ptr(), N, ws.data_ptr(), nbytes, _lib.stream()))
  torch.cuda.synchronize()
  return y


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 256, 256), (1000, 128, 128), (777, 35, 256),
                                   (300, 129, 128), (513, 256, 388), (200, 256, 103), (64, 16, 21),
                                   (5000, 18, 256), (129, 64, 132), (4096, 256, 210)])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_linear_tc_matches_bf16_reference(M, N, K, act):
  torch.manual_seed(M + N + K)
  x = torch.randn(M, K, device=DEV)
  w = torch.randn(N, K, device=DEV) / K ** 0.5
  b = torch.randn(N, device=DEV)
  got = _linear_tc(x, w, b, act)
  ref = (x.bfloat16().double() @ w.bfloat16().double().t() + b.double()).float()
  ref = {0: lambda t: t, 1: torch.nn.functional.elu, 2: torch.relu}[act](ref)
  assert_close_frac("linear_tc", got, ref, rtol=1e-4, atol=1e-4)


def test_linear_tc_is_exact_on_integers():
  """small integers are exact in bf16 and in the fp32 accumulator: bit-exact check
  of the operand layouts / descriptors (any mis-addressed element shows up)."""
  torch.manual_seed(1)
  M, N, K = 384, 256, 320
  x = torch.randint(-4, 5, (M, K), device=DEV).float()
  w = torch.randint(-4, 5, (N, K), device=DEV).float()
  got = _linear_tc(x, w, None, 0)
  assert torch.equal(got, x @ w.t())


@pytest.mark.parametrize("name", ["mv_small", "mono_small", "mono_train"])
def test_bf16_mode_end_to_end(golden, name):
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  fx = golden(name)
  cfg = dict(fx["cfg"])
  cfg["rays"] = 256  # enough rows for the 128-row tensor-core tiles to be exercised
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  d = lambda x: synthetic.to_device(x, DEV)
  with torch.no_grad():
    if cfg["mono"]:
      train = cfg.get("anchor_offset") is not None
      want = orc.render_rays_mono(frame, t, offs, batch, model, feat_c, None, cfg["N_samples"], args,
                                  inv_uniform=True, det=True, is_train=train, num_vv=cfg["num_vv"])
      key = "outputs_coarse_anchor" if train else "outputs_coarse_ref"
    else:
      want = orc.render_rays_mv(frame, t, offs, batch, model, None, feat_c, feat_f, cfg["N_samples"],
                                args, inv_uniform=True, N_importance=cfg["N_importance"], det=True,
                                is_train=False)
      key = "outputs_fine_ref"
  m = synthetic.model_to(model, DEV)
  # per-call precision argument (innermost of the three ways to choose the mode)
  if cfg["mono"]:
    got = rr.render_rays_mono(frame, t, offs, d(batch), m, d(feat_c), Projector(DEV),
                              cfg["N_samples"], args, inv_uniform=True, det=True,
                              is_train=cfg.get("anchor_offset") is not None, num_vv=cfg["num_vv"],
                              precision="bf16")
  else:
    got = rr.render_rays_mv(frame, t, offs, d(batch), m, Projector(DEV), d(feat_c), d(feat_f),
                            cfg["N_samples"], args, inv_uniform=True,
                            N_importance=cfg["N_importance"], det=True, is_train=False, precision="bf16")
  g, w = got[key], want[key]
  # only the stress rigs put samples on in-bounds discontinuities (util.assert_close_frac)
  bad = 0.02 if cfg.get("stress") else 1e-3
  assert_close_frac("rgb", g["rgb"], w["rgb"], rtol=0, atol=2e-3, max_bad_frac=bad)
  assert_close_frac("weights", g["weights"], w["weights"], rtol=0, atol=2e-3, max_bad_frac=bad)
  assert_close_frac("depth", g["depth"], w["depth"], rtol=2e-3, atol=1e-3, max_bad_frac=bad)
  assert orc.psnr(g["rgb"].cpu(), w["rgb"]) > 50.0


# The benchmarked mode at the benchmark's own shapes, against the ORACLE (not the library's fp32 path):
# BASELINE configs[1] (512x288, 64+64 samples, 8+8 views), the view counts eval_nvidia.py really uses
# (7 dynamic + 11 static, eval_nvidia.py:92-119) and the config-4 mono rig (10 dynamic incl. 3 virtual +
# 15 static views).  No stress rig -> no discontinuity allowance beyond 1e-3 of the elements.
BENCH_SHAPES = {
    "bench_8+8": dict(mono=False, H=288, W=512, V_dy=8, V_st=8, rays=96, N_samples=64, N_importance=64, num_vv=0,
                      inv_uniform=True, anti_alias_pooling=1, mask_rgb=0, seed=0, stress=False),
    "nvidia_7+11": dict(mono=False, H=288, W=512, V_dy=7, V_st=11, rays=64, N_samples=64, N_importance=64,
                        num_vv=0, inv_uniform=True, anti_alias_pooling=1, mask_rgb=0, seed=3, stress=False),
    "mono_10+15": dict(mono=True, H=270, W=480, V_dy=10, V_st=15, rays=96, N_samples=64, N_importance=0,
                       num_vv=3, inv_uniform=True, anti_alias_pooling=1, mask_rgb=1, seed=4, stress=False),
}


@pytest.mark.parametrize("name", list(BENCH_SHAPES))
def test_bf16_mode_against_oracle_at_benchmark_shapes(name):
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  cfg = BENCH_SHAPES[name]
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  d = lambda x: synthetic.to_device(x, DEV)
  with torch.no_grad():
    if cfg["mono"]:
      want = orc.render_rays_mono(frame, t, offs, batch, model, feat_c, None, cfg["N_samples"], args,
                                  inv_uniform=True, det=True, is_train=False, num_vv=cfg["num_vv"])
      keys = ("outputs_coarse_ref", "outputs_coarse_ref_dy", "outputs_coarse_st")
    else:
      want = orc.render_rays_mv(frame, t, offs, batch, model, None, feat_c, feat_f, cfg["N_samples"], args,
                                inv_uniform=True, N_importance=cfg["N_importance"], det=True, is_train=False)
      keys = ("outputs_fine_ref", "outputs_fine_ref_dy")
  m = synthetic.model_to(model, DEV)
  rr.set_precision("bf16")
  try:
    if cfg["mono"]:
      got = rr.render_rays_mono(frame, t, offs, d(batch), m, d(feat_c), Projector(DEV), cfg["N_samples"], args,
                                inv_uniform=True, det=True, is_train=False, num_vv=cfg["num_vv"])
    else:
      got = rr.render_rays_mv(frame, t, offs, d(batch), m, Projector(DEV), d(feat_c), d(feat_f),
                              cfg["N_samples"], args, inv_uniform=True, N_importance=cfg["N_importance"],
                              det=True, is_train=False)
  finally:
    rr.set_precision("bf16")
  for key in keys:
    g, w = got[key], want[key]
    for kk in ("rgb", "weights", "depth"):
      err = (g[kk].cpu() - w[kk]).abs().max().item()
      print("%s %s/%s max abs err %.3e" % (name, key, kk, err))
    assert_close_frac(key + "/rgb", g["rgb"], w["rgb"], rtol=0, atol=2e-3, max_bad_frac=1e-3)
    assert_close_frac(key + "/weights", g["weights"], w["weights"], rtol=0, atol=2e-3, max_bad_frac=1e-3)
    assert_close_frac(key + "/depth", g["depth"], w["depth"], rtol=2e-3, atol=1e-3, max_bad_frac=1e-3)
    assert torch.equal(g["mask"].cpu(), w["mask"])
    assert orc.psnr(g["rgb"].cpu(), w["rgb"]) > 50.0


@pytest.mark.parametrize("name", ["mv_small", "mv_linear", "mono_small"])
def test_fused_view_stage_matches_staged(golden, name):
  """The fused per-view kernel (gather + MLP chain + pooling on the tensor cores) against the
  fp32 staged path on the same inputs: raw [R,S,4] of both nets and the projector mask."""
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  fx = golden(name)
  cfg, st = fx["cfg"], fx["stages"]
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  d = lambda x: synthetic.to_device(x, DEV)
  b, fc = d(batch), d(feat_c)
  m = synthetic.model_to(model, DEV)
  pts = d(st["pts"])
  tt = float(t[0].float())
  ray_dir = torch.nn.functional.normalize(b["ray_d"], dim=-1)
  raw_st, m_st = rr.net_static_fused(m.net_coarse_st, pts, b["ray_o"], b["ray_d"], b["camera"],
                                     b["static_src_rgbs"], b["static_src_cameras"],
                                     rr.featmaps_channels_last(fc[2]))
  raw_dy, m_dy = rr.net_dynamic_fused(m.net_coarse_dy, pts, d(st["seq"]), ray_dir, b["camera"],
                                      b["src_rgbs"], b["src_cameras"],
                                      rr.featmaps_channels_last(fc[0]), tt)
  torch.cuda.synchronize()
  assert_close_frac("mask_st", m_st, st["mask_st"], max_bad_frac=1e-3)
  assert_close_frac("mask_dy", m_dy, st["mask_dy"], max_bad_frac=1e-3)
  for br, raw in (("dy", raw_dy), ("st", raw_st)):
    valid = (st["mask_" + br].sum(2) > 0)[..., 0]
    got, want = raw.cpu(), st["raw_" + br]
    assert (got[..., 3][~valid] == -1e9).all()
    assert_close_frac("rgb_" + br, got[..., :3][valid], want[..., :3][valid], rtol=0, atol=1e-2,
                      max_bad_frac=5e-3)
    assert_close_frac("sigma_" + br, got[..., 3][valid], want[..., 3][valid], rtol=0, atol=2e-2,
                      max_bad_frac=5e-3)


def _run_mode(cfg, precision, mono=False):
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  d = lambda x: synthetic.to_device(x, DEV)
  m = synthetic.model_to(model, DEV)
  rr.set_precision(precision)
  try:
    if mono:
      return rr.render_rays_mono(frame, t, offs, d(batch), m, d(feat_c), Projector(DEV), cfg["N_samples"],
                                 args, inv_uniform=True, det=True, is_train=False, num_vv=cfg["num_vv"])
    return rr.render_rays_mv(frame, t, offs, d(batch), m, Projector(DEV), d(feat_c), d(feat_f),
                             cfg["N_samples"], args, inv_uniform=True, N_importance=cfg["N_importance"],
                             det=True, is_train=False)
  finally:
    rr.set_precision("bf16")


def test_wide_view_counts_use_16_slot_kernels():
  """BASELINE config-4 view counts (10 dynamic incl. 3 virtual, 15 static): the fused kernels run
  with 16 view slots per point; compared with the fp32 staged path of the same library."""
  cfg = dict(mono=True, H=36, W=64, V_dy=10, V_st=15, rays=96, N_samples=64, N_importance=0, num_vv=3,
             inv_uniform=True, anti_alias_pooling=1, mask_rgb=1, seed=31, stress=True)
  ref = _run_mode(cfg, "fp32", mono=True)["outputs_coarse_ref"]
  got = _run_mode(cfg, "bf16", mono=True)["outputs_coarse_ref"]
  assert_close_frac("rgb", got["rgb"], ref["rgb"], rtol=0, atol=2e-3, max_bad_frac=0.03)
  assert_close_frac("weights", got["weights"], ref["weights"], rtol=0, atol=2e-3, max_bad_frac=0.03)
  assert torch.equal(got["mask"], ref["mask"])


def test_config4_sample_counts_use_simt_attention_for_192_samples():
  """BASELINE config-4 sample counts (64 coarse + 128 importance -> the fine pass evaluates 192 samples per
  ray, 10 source views): 192 does not divide the 128-row attention tile, so the ray transformer runs in the
  SIMT kernel on the bf16 tile images; compared with the fp32 staged path of the same library."""
  cfg = dict(mono=False, H=36, W=64, V_dy=10, V_st=10, rays=48, N_samples=64, N_importance=128, num_vv=0,
             inv_uniform=True, anti_alias_pooling=1, mask_rgb=0, seed=33, stress=False)
  ref = _run_mode(cfg, "fp32")["outputs_fine_ref"]
  got = _run_mode(cfg, "bf16")["outputs_fine_ref"]
  assert got["weights"].shape[-1] == 192
  assert_close_frac("rgb", got["rgb"], ref["rgb"], rtol=0, atol=2e-3, max_bad_frac=1e-3)
  assert_close_frac("weights", got["weights"], ref["weights"], rtol=0, atol=2e-3, max_bad_frac=1e-3)


def test_more_than_16_views_falls_back_to_staged_tensor_core_layers():
  cfg = dict(mono=False, H=36, W=64, V_dy=7, V_st=18, rays=64, N_samples=16, N_importance=16, num_vv=0,
             inv_uniform=True, anti_alias_pooling=1, mask_rgb=0, seed=32, stress=False)
  ref = _run_mode(cfg, "fp32")["outputs_fine_ref"]
  got = _run_mode(cfg, "bf16")["outputs_fine_ref"]
  assert_close_frac("rgb", got["rgb"], ref["rgb"], rtol=0, atol=2e-3, max_bad_frac=1e-3)


@pytest.mark.parametrize("rays", [0, 1, 255, 257])
def test_ragged_and_empty_ray_batches(rays):
  """empty / single-ray / non-multiple-of-tile batches through the fused path."""
  cfg = dict(scenes.GOLDEN_CONFIGS["mv_small"], rays=max(rays, 1), N_samples=32, N_importance=32)
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  if rays == 0:
    for k in ("ray_o", "ray_d", "uv_grid"):
      batch[k] = batch[k][:0]
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  want = None
  if rays:  # oracle first: model_to() below moves the modules to the GPU in place
    with torch.no_grad():
      want = orc.render_rays_mv(frame, t, offs, batch, model, None, feat_c, feat_f, 32, args,
                                inv_uniform=True, N_importance=32, det=True, is_train=False)["outputs_fine_ref"]
  d = lambda x: synthetic.to_device(x, DEV)
  m = synthetic.model_to(model, DEV)
  rr.set_precision("bf16")
  try:
    got = rr.render_rays_mv(frame, t, offs, d(batch), m, Projector(DEV), d(feat_c), d(feat_f), 32, args,
                            inv_uniform=True, N_importance=32, det=True, is_train=False)["outputs_fine_ref"]
  finally:
    rr.set_precision("bf16")
  assert got["rgb"].shape == (rays, 3) and got["weights"].shape == (rays, 64)
  if rays:
    assert_close_frac("rgb", got["rgb"], want["rgb"], rtol=0, atol=2e-3, max_bad_frac=0.03)


def test_bf16_full_size_properties():
  """BASELINE config-2 chunk (8192 rays, 64+64 samples, 8+8 views, 512x288) in the benchmarked
  mode: rays are independent -> permuting the rays permutes the outputs bit-exactly; weights are
  a sub-probability distribution; depths sorted; parity with the fp32 path on a sub-sample."""
  cfg = dict(mono=False, H=288, W=512, V_dy=8, V_st=8, rays=8192, N_samples=64, N_importance=64,
             num_vv=0, inv_uniform=True, anti_alias_pooling=1, mask_rgb=0, seed=21, stress=False)
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  d = lambda x: synthetic.to_device(x, DEV)
  b, fc, ff = d(batch), d(feat_c), d(feat_f)
  m = synthetic.model_to(model, DEV)

  def run(bb, prec):
    rr.set_precision(prec)
    try:
      return rr.render_rays_mv(frame, t, offs, bb, m, Projector(DEV), fc, ff, 64, args, inv_uniform=True,
                               N_importance=64, det=True, is_train=False)["outputs_fine_ref"]
    finally:
      rr.set_precision("bf16")

  full = run(b, "bf16")
  perm = torch.randperm(8192, device=DEV)
  bp = dict(b)
  for k in ("ray_o", "ray_d", "uv_grid"):
    bp[k] = b[k][perm].contiguous()
  permuted = run(bp, "bf16")
  for k in ("rgb", "depth", "weights"):
    assert torch.equal(permuted[k], full[k][perm]), k
  w = full["weights"]
  assert torch.isfinite(full["rgb"]).all() and (w >= 0).all() and (w.sum(1) <= 1 + 1e-3).all()
  assert (full["z_vals"][:, 1:] >= full["z_vals"][:, :-1]).all()
  sub = dict(b)
  for k in ("ray_o", "ray_d", "uv_grid"):
    sub[k] = b[k][:512].contiguous()
  ref = run(sub, "fp32")
  assert_close_frac("rgb", full["rgb"][:512], ref["rgb"], rtol=0, atol=2e-3, max_bad_frac=1e-3)
  assert orc.psnr(full["rgb"][:512].cpu(), ref["rgb"].cpu()) > 50.0
