"""Multi-camera ray batches: the K target cameras of one time step rendered in one pass
(sample_ray.stack_ray_batches, render_image.render_multi_image_nvi, dyn_net_static_fused_mc,
dyn_project_gather_mc).

Rays are independent, so every output of a camera rendered inside a multi-camera batch must equal, bit for bit,
the same camera rendered alone by render_single_image_nvi -- in both precisions, with chunks that straddle the
camera boundaries.  Permuting camera_index must change the static branch (its ray_diff reads the target camera)
and leave the dynamic net's output alone.  One mixed chunk is checked per camera against the CPU oracle at the
DESIGN.md §2 bars, and the unsupported uses fail loudly.
"""

import pytest
import torch

import scenes
from dynibar_b200 import _lib, synthetic
from dynibar_b200 import render_ray as rr
from dynibar_b200 import sample_ray as sr
from dynibar_b200.projection import Projector
from dynibar_b200.render_image import render_multi_image_nvi, render_single_image_nvi
from oracle import dynibar_oracle as orc
from util import assert_close_frac

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H, W = 48, 96
# three target cameras at distinct centres around the make_cameras rig (whose target sits at the origin)
TARGET_OFFSETS = ((0.0, 0.0, 0.0), (0.045, 0.012, -0.02), (-0.03, -0.017, 0.035))


def _scene(V_st, seed=21):
  cfg = dict(scenes.GOLDEN_CONFIGS["mv_small"], H=H, W=W, V_st=V_st, rays=None, seed=seed, stress=False)
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  assert args.anti_alias_pooling == 1
  data = scenes.sampler_data(batch, H, W, cfg["seed"])
  K_mat = sr.parse_camera(batch["camera"])[2][0]
  samplers = []
  for off in TARGET_OFFSETS:
    c2w = torch.eye(4)
    c2w[:3, 3] = torch.tensor(off)
    samplers.append(sr.RaySamplerSingleImage(dict(data, camera=synthetic.camera_vector(H, W, K_mat, c2w)[None]), DEV))
  return cfg, samplers, feat_c, feat_f, frame, t, offs, model, args


@pytest.fixture(scope="module", params=[5, 11], ids=["V_st5", "V_st11"])
def scene(request):
  cfg, samplers, feat_c, feat_f, frame, t, offs, model, args = _scene(request.param)
  dev = lambda x: synthetic.to_device(x, DEV)
  return dict(cfg=cfg, samplers=samplers, fc=dev(feat_c), ff=dev(feat_f), frame=frame, t=t, offs=offs,
              model=synthetic.model_to(model, DEV), args=args)


def _render_multi(s, batch, chunk, precision):
  with rr.precision_scope(precision):
    return render_multi_image_nvi(s["frame"], s["t"], s["offs"], s["samplers"], batch, s["model"], Projector(DEV),
                                  chunk, s["cfg"]["N_samples"], s["args"], inv_uniform=s["cfg"]["inv_uniform"],
                                  N_importance=s["cfg"]["N_importance"], det=True, coarse_featmaps=s["fc"],
                                  fine_featmaps=s["ff"], is_train=False)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_multi_camera_render_equals_single_camera_renders_bitwise(scene, precision):
  s = scene
  batch, counts, hw = sr.stack_ray_batches([smp.get_all() for smp in s["samplers"]])
  assert counts == [H * W] * 3 and hw == (H, W)
  chunk = 1000  # divides neither a camera's 4608 rays nor the batch's 13824: chunks straddle cameras
  multi = _render_multi(s, batch, chunk, precision)
  assert len(multi) == 3
  for k, smp in enumerate(s["samplers"]):
    with rr.precision_scope(precision):
      single = render_single_image_nvi(s["frame"], s["t"], s["offs"], smp, smp.get_all(), s["model"],
                                       Projector(DEV), chunk, s["cfg"]["N_samples"], s["args"],
                                       inv_uniform=s["cfg"]["inv_uniform"], N_importance=s["cfg"]["N_importance"],
                                       det=True, coarse_featmaps=s["fc"], fine_featmaps=s["ff"], is_train=False)
    got = multi[k]
    assert list(got.keys()) == list(single.keys()) and got["outputs_fine"] is None
    assert len(got["outputs_fine_anchor"]) == 0
    for name in ("outputs_fine_ref", "outputs_coarse_ref"):
      assert list(got[name].keys()) == list(single[name].keys()), name
      for key, want in single[name].items():
        g = got[name][key]
        assert not g.is_cuda and g.shape == want.shape and g.dtype == want.dtype, (k, name, key)
        assert torch.equal(g, want), "camera %d %s/%s differs from the single-camera render" % (k, name, key)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_permuted_camera_index_changes_the_static_branch_only(scene, precision):
  s = scene
  batch, _, _ = sr.stack_ray_batches([smp.get_all() for smp in s["samplers"]])
  ref = _render_multi(s, batch, 4096, precision)
  perm = dict(batch, camera_index=((batch["camera_index"] + 1) % 3).to(torch.int32))
  got = _render_multi(s, perm, 4096, precision)
  for k in range(3):
    a, b = got[k]["outputs_coarse_ref"], ref[k]["outputs_coarse_ref"]
    # ray_diff drives the static net's anti-alias pooling weights and its blending head
    assert not torch.equal(a["rgb_static"], b["rgb_static"]), k
    assert not torch.equal(a["rgb"], b["rgb"]), k
    # the dynamic net discards ray_diff: its alphas stay (rgb_dy and weights_dy composite with the joint
    # transmittance, which includes the static density)
    assert torch.equal(a["alpha_dy"], b["alpha_dy"]), k


def test_mixed_chunk_against_oracle_per_camera():
  cfg, samplers, feat_c, feat_f, frame, t, offs, model, args = _scene(11, seed=22)
  g = torch.Generator().manual_seed(5)
  parts = []
  for smp in samplers:
    b = smp.get_all()
    sel = torch.randperm(H * W, generator=g)[:48].to(DEV)
    parts.append(dict(b, ray_o=b["ray_o"][sel], ray_d=b["ray_d"][sel], uv_grid=b["uv_grid"][sel]))
  batch, counts, _ = sr.stack_ray_batches(parts)
  mix = torch.randperm(sum(counts), generator=g)  # cameras interleaved inside the chunk
  for key in ("ray_o", "ray_d", "uv_grid", "camera_index"):
    batch[key] = batch[key][mix.to(DEV)]
  where = torch.argsort(mix)  # where[i]: position of stacked ray i in the mixed chunk
  # oracle first: model_to() below moves the modules to the GPU in place
  want = []
  for p in parts:
    cpu = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in p.items()}
    with torch.no_grad():
      want.append(orc.render_rays_mv(frame, t, offs, cpu, model, None, feat_c, feat_f, cfg["N_samples"], args,
                                     inv_uniform=cfg["inv_uniform"], N_importance=cfg["N_importance"], det=True,
                                     is_train=False)["outputs_fine_ref"])
  m_dev = synthetic.model_to(model, DEV)
  fc, ff = synthetic.to_device(feat_c, DEV), synthetic.to_device(feat_f, DEV)
  for precision in ("bf16", "fp32"):
    got = rr.render_rays_mv(frame, t, offs, batch, m_dev, Projector(DEV), fc, ff, cfg["N_samples"], args,
                            inv_uniform=cfg["inv_uniform"], N_importance=cfg["N_importance"], det=True,
                            is_train=False, precision=precision)["outputs_fine_ref"]
    for k, w in enumerate(want):
      pick = where[sum(counts[:k]):sum(counts[:k + 1])].to(DEV)
      gk = {key: got[key][pick].cpu() for key in ("rgb", "weights", "depth")}
      tag = "%s camera %d " % (precision, k)
      if precision == "bf16":
        assert_close_frac(tag + "rgb", gk["rgb"], w["rgb"], rtol=0, atol=2e-3, max_bad_frac=1e-3)
        assert_close_frac(tag + "weights", gk["weights"], w["weights"], rtol=0, atol=2e-3, max_bad_frac=1e-3)
        assert_close_frac(tag + "depth", gk["depth"], w["depth"], rtol=2e-3, atol=1e-3, max_bad_frac=1e-3)
        assert orc.psnr(gk["rgb"], w["rgb"]) > 50.0
      else:
        for key in ("rgb", "weights", "depth"):
          assert_close_frac(tag + key, gk[key], w[key], rtol=5e-4, atol=5e-5, max_bad_frac=1e-3)


def _small_multi_batch(s, n=32):
  parts = []
  for smp in s["samplers"]:
    b = smp.get_all()
    parts.append(dict(b, ray_o=b["ray_o"][:n], ray_d=b["ray_d"][:n], uv_grid=b["uv_grid"][:n]))
  return sr.stack_ray_batches(parts)[0]


def _mv(s, batch, precision="bf16"):
  return rr.render_rays_mv(s["frame"], s["t"], s["offs"], batch, s["model"], Projector(DEV), s["fc"], s["ff"],
                           s["cfg"]["N_samples"], s["args"], inv_uniform=True, N_importance=s["cfg"]["N_importance"],
                           det=True, is_train=False, precision=precision)


def test_unsupported_multi_camera_uses_fail_loudly(scene):
  s = scene
  batch = _small_multi_batch(s)
  # 17 target cameras: the Python entry refuses, and so does the C ABI
  b17 = dict(batch, camera=batch["camera"][[0] * 17])
  with pytest.raises(ValueError, match="at most 16"):
    _mv(s, b17)
  # K > 1 without a per-ray camera index
  with pytest.raises(ValueError, match="camera_index"):
    _mv(s, {k: v for k, v in batch.items() if k != "camera_index"})
  # a camera_index outside [0, K) is caught once per frame, before any rendering
  full, _, _ = sr.stack_ray_batches([smp.get_all() for smp in s["samplers"]])
  bad = dict(full, camera_index=full["camera_index"] + 1)
  with pytest.raises(ValueError, match="camera_index spans"):
    render_multi_image_nvi(s["frame"], s["t"], s["offs"], s["samplers"], bad, s["model"], Projector(DEV), 1000,
                           s["cfg"]["N_samples"], s["args"], N_importance=s["cfg"]["N_importance"], det=True,
                           coarse_featmaps=s["fc"], fine_featmaps=s["ff"], is_train=False)
  # the twin-warp per-view kernel has no multi-camera form
  _lib.lib.dyn_debug_set_view_kernel(0)
  try:
    with pytest.raises(RuntimeError, match="twin-warp"):
      _mv(s, batch, "bf16")
  finally:
    _lib.lib.dyn_debug_set_view_kernel(-1)
  # monocular rendering and training stay single-camera
  args = s["args"]
  with pytest.raises(NotImplementedError, match="multi-camera"):
    rr.render_rays_mono(s["frame"], s["t"], s["offs"], batch, s["model"], s["fc"], Projector(DEV),
                        s["cfg"]["N_samples"], args, inv_uniform=True, det=True, is_train=False)
  net = s["model"].net_coarse_st
  net.requires_grad_(True)
  try:
    with torch.enable_grad(), pytest.raises(NotImplementedError, match="multi-camera"):
      rr.render_rays_mono(s["frame"], s["t"], s["offs"], batch, s["model"], s["fc"], Projector(DEV),
                          s["cfg"]["N_samples"], args, inv_uniform=True, det=True, is_train=True)
  finally:
    net.requires_grad_(False)
