"""Pooled multi-camera monocular rendering (sample_ray.stack_pooled_ray_batches,
render_image.render_multi_image_mono, the *_tbl entry points): the target cameras of one time step, each with its
own source views drawn from shared pools, rendered in one pass.

Rays are independent and a camera's slot v reads pool entry table[k][v], so every output of camera k inside the
pooled batch must equal, bit for bit, render_single_image_mono on camera k alone with its views sliced from the
pools (pool[table[k]], feature maps included) -- fused bf16 (VP 16 and VP 8), fp32 staged and bf16 staged
(17-32 static slots), K = 1, 3 and 16, pools of exactly 16 and 32, a pool entry no camera uses, cameras whose
virtual views come in different orders, and chunks that straddle cameras (except on the staged bf16 networks, whose
results depend in the last bits on which rays share a call).
"""

import pytest
import torch

import scenes
from dynibar_b200 import _lib, synthetic
from dynibar_b200 import render_ray as rr
from dynibar_b200 import sample_ray as sr
from dynibar_b200.projection import Projector, project_gather
from dynibar_b200.render_image import render_multi_image_mono, render_single_image_mono

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_SAMPLES = 32


def _offsets(K):
  g = torch.Generator().manual_seed(K)
  return [(0.0, 0.0, 0.0)] + [tuple((0.08 * (torch.rand(3, generator=g) - 0.5)).tolist()) for _ in range(K - 1)]


def _plan(K, n_t, n_vv, vv_pool, n_st, st_pool, seed):
  """Per camera: dynamic identities (temporal frames 0..n_t-1, then n_vv virtual views in a camera-specific order)
  and n_st static frames, drawn round-robin from pools of vv_pool virtual and st_pool static views so that every
  pool entry is used (the builder keeps used views only)."""
  assert K * n_vv >= vv_pool and K * n_st >= st_pool
  g = torch.Generator().manual_seed(seed)
  dy, st = [], []
  for k in range(K):
    vv = [(k * n_vv + i) % vv_pool for i in range(n_vv)]
    dy.append(list(range(n_t)) + [("vv", vv[i]) for i in torch.randperm(n_vv, generator=g).tolist()])
    st.append(sorted((k * n_st + i) % st_pool for i in range(n_st)))
  return dy, st


def _scene(K, H, W, n_t, n_vv, vv_pool, n_st, st_pool, seed=31, extra_static=False):
  cfg = dict(scenes.GOLDEN_CONFIGS["mono_small"], H=H, W=W, V_dy=n_t + vv_pool, V_st=st_pool, rays=None, seed=seed,
             stress=False, N_samples=N_SAMPLES, num_vv=n_vv)
  batch, feat_c, _, frame, t, _, model, args = scenes.build(cfg)
  offs = (synthetic.time_offsets(n_t + n_vv, n_vv), None)
  data = scenes.sampler_data(batch, H, W, seed)
  K_mat = sr.parse_camera(batch["camera"])[2][0]
  dy_ids, st_ids = _plan(K, n_t, n_vv, vv_pool, n_st, st_pool, seed)
  dy_at = lambda ident: ident if not isinstance(ident, tuple) else n_t + ident[1]  # index into the scene's views
  samplers, parts, feats = [], [], []
  for k, off in enumerate(_offsets(K)):
    c2w = torch.eye(4)
    c2w[:3, 3] = torch.tensor(off)
    smp = sr.RaySamplerSingleImage(dict(data, camera=synthetic.camera_vector(H, W, K_mat, c2w)[None]), DEV)
    di = torch.tensor([dy_at(i) for i in dy_ids[k]])
    si = torch.tensor(st_ids[k])
    b = smp.get_all()
    b["src_rgbs"], b["src_cameras"] = batch["src_rgbs"][:, di].to(DEV), batch["src_cameras"][:, di].to(DEV)
    b["static_src_rgbs"] = batch["static_src_rgbs"][:, si].to(DEV)
    b["static_src_cameras"] = batch["static_src_cameras"][:, si].to(DEV)
    samplers.append(smp)
    parts.append(b)
    feats.append((feat_c[0][di].to(DEV), None, feat_c[2][si].to(DEV)))
  pooled, counts, hw = sr.stack_pooled_ray_batches(parts, dy_ids, st_ids)
  assert hw == (H, W) and counts == [H * W] * K
  pool_feats = (feat_c[0][[dy_at(i) for i in pooled["src_view_ids"]]].to(DEV), None,
                feat_c[2][pooled["static_src_view_ids"]].to(DEV))
  if extra_static:  # a pool entry no camera uses: appended, the tables unchanged
    g = torch.Generator().manual_seed(seed + 1)
    pooled["static_src_rgbs"] = torch.cat([pooled["static_src_rgbs"],
                                           torch.rand(1, 1, H, W, 3, generator=g).to(DEV)], 1)
    cam = pooled["static_src_cameras"][:, :1].clone()
    cam[0, 0, 18 + 3] += 0.3
    pooled["static_src_cameras"] = torch.cat([pooled["static_src_cameras"], cam], 1)
    pool_feats = (pool_feats[0], None, torch.cat([pool_feats[2], torch.randn(1, *pool_feats[2].shape[1:],
                                                                             generator=g).to(DEV)]))
  return dict(samplers=samplers, parts=parts, feats=feats, pooled=pooled, pool_feats=pool_feats, frame=frame, t=t,
              offs=offs, model=synthetic.model_to(model, DEV), args=args, num_vv=n_vv, K=K)


def _render_single(s, k, chunk, precision):
  with rr.precision_scope(precision):
    return render_single_image_mono(s["frame"], s["t"], s["offs"], s["samplers"][k], s["parts"][k], s["model"],
                                    Projector(DEV), chunk, N_SAMPLES, s["args"], inv_uniform=True, det=True,
                                    featmaps=s["feats"][k], is_train=False, num_vv=s["num_vv"])


def _render_multi(s, chunk, precision):
  with rr.precision_scope(precision):
    return render_multi_image_mono(s["frame"], s["t"], s["offs"], s["samplers"], s["pooled"], s["model"],
                                   Projector(DEV), chunk, N_SAMPLES, s["args"], inv_uniform=True, det=True,
                                   featmaps=s["pool_feats"], is_train=False, num_vv=s["num_vv"])


def _assert_bitwise(got, want):
  assert list(got.keys()) == list(want.keys()) and got["outputs_fine"] is None
  assert len(got["outputs_coarse_anchor"]) == 0 and len(want["outputs_coarse_anchor"]) == 0
  for name in ("outputs_coarse_ref", "outputs_coarse_st"):
    assert list(got[name].keys()) == list(want[name].keys()), name
    for key, w in want[name].items():
      g = got[name][key]
      assert g.shape == w.shape and g.dtype == w.dtype, (name, key)
      assert torch.equal(g, w), (name, key, (g.float() - w.float()).abs().max().item())


# (name, precision, K, H, W, temporal, vv slots, vv pool, static slots, static pool, extra static entry, chunk)
CASES = [
    ("fused_vp16", "bf16", 3, 24, 40, 7, 3, 8, 15, 20, False, 700),
    ("fused_vp8", "bf16", 3, 24, 40, 6, 2, 5, 8, 12, True, 500),
    ("fp32_staged", "fp32", 3, 24, 40, 7, 3, 8, 15, 20, False, 700),
    # chunks of one camera's rays: the staged bf16 networks (17-32 slots) are not bit-for-bit invariant to which
    # rays share a network call, with or without tables (chunks across cameras move the rgb by ~5e-5)
    ("bf16_staged_st20_pool32", "bf16", 3, 24, 40, 7, 3, 8, 20, 32, False, 24 * 40),
    ("k1", "bf16", 1, 24, 40, 7, 3, 3, 15, 15, False, 700),
    ("k16_pool16", "bf16", 16, 8, 12, 7, 3, 9, 15, 16, False, 250),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_pooled_render_equals_single_camera_renders_bitwise(case):
  name, prec, K, H, W, n_t, n_vv, vv_pool, n_st, st_pool, extra, chunk = case
  s = _scene(K, H, W, n_t, n_vv, vv_pool, n_st, st_pool, extra_static=extra)
  p = s["pooled"]
  assert p["src_cameras"].shape[1] == n_t + vv_pool
  assert p["static_src_cameras"].shape[1] == st_pool + extra
  if K > 1:  # the cameras' virtual views come in different orders
    assert len({tuple(r[n_t:]) for r in p["src_views"].tolist()}) > 1
  multi = _render_multi(s, chunk, prec)
  assert len(multi) == K
  for k in range(K):
    _assert_bitwise(multi[k], _render_single(s, k, chunk, prec))


def test_table_kernels_equal_single_camera_calls_on_sliced_views():
  """dyn_project_gather_tbl and dyn_plucker_src_tbl against dyn_project_gather / dyn_plucker_src on each
  camera's own views, on that camera's rays."""
  s = _scene(3, 16, 24, 7, 3, 8, 20, 32, seed=41)
  p = s["pooled"]
  dev_rays = p["ray_o"].shape[0]
  g = torch.Generator().manual_seed(3)
  pts = (torch.randn(dev_rays, 8, 3, generator=g) * 0.5 + torch.tensor([0.0, 0.0, 4.0])).to(DEV)
  V = p["static_src_views"].shape[1]
  ci = p["camera_index"]
  cams = p["camera"]
  f_all, rd_all, m_all = project_gather(pts, None, cams, p["static_src_rgbs"], p["static_src_cameras"],
                                        s["pool_feats"][2], ci, p["static_src_views"])
  pl_all = rr.compute_src_plucker_coordinate(pts, p["static_src_cameras"], ci, p["static_src_views"])
  lo = 0
  for k, part in enumerate(s["parts"]):
    n = part["ray_o"].shape[0]
    f, rd, m = project_gather(pts[lo:lo + n], None, part["camera"], part["static_src_rgbs"],
                              part["static_src_cameras"], s["feats"][k][2])
    pl = rr.compute_src_plucker_coordinate(pts[lo:lo + n], part["static_src_cameras"])
    assert f.shape[2] == V
    for got, want in ((f_all, f), (rd_all, rd), (m_all, m), (pl_all, pl)):
      assert torch.equal(got[lo:lo + n], want)
    lo += n


def test_pooled_uses_that_stay_unsupported_fail_loudly():
  s = _scene(3, 8, 12, 7, 3, 8, 15, 20)
  p = s["pooled"]
  with pytest.raises(NotImplementedError, match="multi-camera"):
    rr.render_rays_mono(s["frame"], s["t"], s["offs"], p, s["model"], s["pool_feats"], Projector(DEV), N_SAMPLES,
                        s["args"], inv_uniform=True, det=True, is_train=True, num_vv=s["num_vv"])
  with pytest.raises(NotImplementedError, match="is_train=False"):
    render_multi_image_mono(s["frame"], s["t"], s["offs"], s["samplers"], p, s["model"], Projector(DEV), 100,
                            N_SAMPLES, s["args"], inv_uniform=True, det=True, featmaps=s["pool_feats"], is_train=True,
                            num_vv=s["num_vv"])
  bad = dict(p, static_src_views=p["static_src_views"] + 5)
  with pytest.raises(ValueError, match="static_src_views spans"):
    render_multi_image_mono(s["frame"], s["t"], s["offs"], s["samplers"], bad, s["model"], Projector(DEV), 100,
                            N_SAMPLES, s["args"], inv_uniform=True, det=True, featmaps=s["pool_feats"],
                            num_vv=s["num_vv"])
  # the twin-warp per-view kernel has no table form
  _lib.lib.dyn_debug_set_view_kernel(0)
  try:
    with pytest.raises(RuntimeError, match="twin-warp"):
      with rr.precision_scope("bf16"):
        render_multi_image_mono(s["frame"], s["t"], s["offs"], s["samplers"], p, s["model"], Projector(DEV), 100,
                                N_SAMPLES, s["args"], inv_uniform=True, det=True, featmaps=s["pool_feats"],
                                num_vv=s["num_vv"])
  finally:
    _lib.lib.dyn_debug_set_view_kernel(-1)
