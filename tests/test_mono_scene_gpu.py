"""The device-resident monocular scene (dynibar_b200.mono_scene, csrc/scene.cu) on the GPU:
  - against the reference's own loader (tests/golden/mono_scene.pt, make_golden_scene.py), bit for bit: ids, source
    stacks, target rgb / masks / flows, rays' supervision and uv; disparity, cameras and depth range within one
    float32 ulp (the fixture was recorded under numpy 2, whose float32 `scale` can differ from the reference
    environment's by one ulp); ray_o / ray_d within RAY_BAR;
  - the mask kernels against tests/mono_scene_ref.py (cv2 + scipy) at 288x512 and odd sizes, bit for bit;
  - `sample` repeats bit for bit and makes no synchronising call;
  - a training step fed from the scene gives the loss of the same step fed the host path's batch."""

import io
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import mono_scene_ref as msr

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mono_scene.pt")
# ray_d against the reference's float32 host bmm (M [u, v, 1] in another summation order): 2x the worst measured on the
# fixture, 1.19e-7 (the kernel's arithmetic is IEEE fp32 without contraction, so the host evaluation of the same
# expression in tests/test_mono_scene_host_cpu.py measures the same number)
RAY_BAR = 2.4e-7


def _camera_close(a, b):
  """[..., 34] cameras: size and intrinsics equal; rotation and translation within one float32 ulp of their largest
  entry (numpy 2's float32 scale moves the centres and, through the mean camera, the recentred rotations)."""
  a, b = a.detach().cpu(), b.detach().cpu()
  assert a.shape == b.shape and torch.equal(a[..., :18], b[..., :18])
  ra, rb = a[..., 18:34].reshape(-1, 4, 4), b[..., 18:34].reshape(-1, 4, 4)
  eps = torch.finfo(torch.float32).eps
  for blk in (np.s_[:, :3, :3], np.s_[:, :3, 3]):
    assert (ra[blk] - rb[blk]).abs().max() <= eps * rb[blk].abs().max()


def _ulp_close(a, b, ulps=1):
  a, b = a.detach().cpu().float(), b.detach().cpu().float()
  assert a.shape == b.shape, (a.shape, b.shape)
  tol = ulps * torch.finfo(torch.float32).eps * torch.maximum(a.abs(), b.abs())
  assert ((a - b).abs() <= tol).all(), ((a - b).abs() - tol).max().item()


@pytest.fixture(scope="module")
def golden():
  return msr.load_golden(GOLDEN)


@pytest.fixture(scope="module")
def raws(golden):
  return {name: dict(np.load(io.BytesIO(sc["raw"]))) for name, sc in golden["scenes"].items()}


@pytest.fixture(scope="module")
def scene_dirs(raws, tmp_path_factory):
  root = tmp_path_factory.mktemp("mono_scene")
  return {name: msr.write_scene(str(root / name / "dense"), raw) for name, raw in raws.items()}


def _args(golden, case):
  sc = golden["scenes"][case["scene"]]
  return SimpleNamespace(training_height=sc["height"], mask_src_view=case["mask_src_view"],
                         erosion_radius=case["erosion_radius"], **golden["base"])


def test_sample_matches_reference_loader(golden, raws, scene_dirs):
  from dynibar_b200 import mono_scene, sample_ray
  dev = torch.device("cuda:0")
  scenes = {}
  for c in golden["cases"]:
    key = (c["scene"], c["mask_src_view"], c["erosion_radius"])
    if key not in scenes:
      scenes[key] = mono_scene.MonocularScene(scene_dirs[c["scene"]], _args(golden, c), dev)
    s = scenes[key]
    s.set_epoch(c["epoch"])
    sample_ray.rng = np.random.RandomState(c["pixel_seed"])
    td, rb = s.sample(np.random.RandomState(c["seed"]), golden["n_rand"], c["sample_mode"])
    torch.cuda.synchronize()
    what = "%s seed %d epoch %d" % (key, c["seed"], c["epoch"])
    for k in ("id", "anchor_id", "num_frames", "ref_time", "anchor_time", "nearest_pose_ids",
              "anchor_nearest_pose_ids"):
      assert td[k].dtype == c[k].dtype and torch.equal(td[k].cpu(), c[k]), (what, k)
    for k, (dt, shape) in c["dtypes"].items():
      assert str(td[k].dtype) == dt and tuple(td[k].shape) == shape and td[k].is_cuda, (what, k)
    assert os.path.relpath(td["rgb_path"][0], s.scene_path) == c["rgb_path"]
    for k in ("motion_mask", "static_mask"):
      assert torch.equal(td[k].cpu(), torch.from_numpy(msr.unpack_mask(c[k]))[None]), (what, k)
    for k, h in c["hash"].items():
      if k != "disp":  # within one ulp: below
        assert msr.hash_f32(td[k]) == h, (what, k)
    for k in ("camera", "anchor_camera", "src_cameras", "static_src_cameras", "anchor_src_cameras"):
      _camera_close(td[k], c[k])
    _ulp_close(td["depth_range"], c["depth_range"])
    # the fixture's disparity is the raw disparity / its float32 scale (tests/test_mono_scene_reference_cpu.py)
    sc = golden["scenes"][c["scene"]]
    _ulp_close(td["disp"], torch.from_numpy(raws[c["scene"]]["disp"][int(c["id"])] / np.float32(sc["scale"]))[None])
    assert sorted(rb) == c["ray_keys"], what
    r = c["rays"]
    assert np.array_equal(rb["selected_inds"], r["selected_inds"].numpy()), what
    for k in ("rgb", "motion_mask", "static_mask", "uv_grid", "flows", "masks"):
      assert torch.equal(rb[k].cpu(), r[k]), (what, k)
    _ulp_close(rb["disp"], r["disp"])
    t = c["camera"][0, 18:34].reshape(4, 4)[:3, 3]
    assert (rb["ray_o"].cpu() - r["ray_o"]).abs().max() <= torch.finfo(torch.float32).eps * t.abs().max()
    err = (rb["ray_d"].cpu() - r["ray_d"]).abs().max().item()
    print("%s: ray_d max abs err vs the reference's bmm %.3e" % (what, err))
    assert err <= RAY_BAR, (what, err)
    for k in ("src_rgbs", "static_src_rgbs", "anchor_src_rgbs", "src_cameras", "camera"):
      assert rb[k] is td[k]


def _run_masks(dyn, st, H, W, radius):
  from dynibar_b200 import _lib
  dev = torch.device("cuda:0")
  n = dyn.shape[0]
  mc = 1 if dyn.ndim == 3 else dyn.shape[-1]
  eh, ew = msr.ERODE_H, int(round(msr.ERODE_H * W / H))
  d = torch.from_numpy(np.ascontiguousarray(dyn)).to(dev)
  s = torch.from_numpy(np.ascontiguousarray(st)).to(dev)
  motion = torch.empty(n, H, W, dtype=torch.uint8, device=dev)
  stat = torch.empty_like(motion)
  src = torch.empty(n, H, W, mc, dtype=torch.uint8, device=dev)
  ws = torch.empty(_lib.lib.dyn_scene_masks_workspace_bytes(n, eh, ew), dtype=torch.uint8, device=dev)
  _lib.check(_lib.lib.dyn_scene_masks(d.data_ptr(), dyn.shape[1], dyn.shape[2], mc, s.data_ptr(), st.shape[1],
                                      st.shape[2], n, H, W, eh, ew, radius, motion.data_ptr(), stat.data_ptr(),
                                      src.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream()))
  return motion.cpu().numpy(), stat.cpu().numpy(), src.cpu().numpy()


@pytest.mark.parametrize("H,W,mh,mw", msr.MASK_SIZES)
@pytest.mark.parametrize("channels", [0, 3])
def test_mask_kernels_match_restatement(H, W, mh, mw, channels):
  for kind, dyn, st in msr.mask_inputs(H, W, mh, mw, channels):
    for r in range(6):
      motion, stat, src = _run_masks(dyn, st, H, W, r)
      for i in range(len(dyn)):
        np.testing.assert_array_equal(motion[i], msr.motion_mask(dyn[i], H, W, r), err_msg="%s r=%d" % (kind, r))
        if r == 0:
          np.testing.assert_array_equal(stat[i], msr.static_mask(st[i], H, W))
          got = src[i].astype(np.float32) / np.float32(255.0)
          np.testing.assert_array_equal(got, msr.source_mask(dyn[i], H, W))


def test_sample_is_repeatable_and_does_not_synchronise(golden, scene_dirs):
  from dynibar_b200 import mono_scene, sample_ray
  c = golden["cases"][0]
  s = mono_scene.MonocularScene(scene_dirs[c["scene"]], _args(golden, c), torch.device("cuda:0"))
  s.set_epoch(3)
  outs = []
  for _ in range(2):
    sample_ray.rng = np.random.RandomState(5)
    rng = np.random.RandomState(9)
    got = []
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
      for _ in range(6):  # more steps than staging buffers
        got.append(s.sample(rng, 128, "uniform"))
    finally:
      torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    outs.append(got)
  for (ta, ra), (tb, rbb) in zip(*outs):
    for a, b in ((ta, tb), (ra, rbb)):
      assert sorted(a) == sorted(b)
      for k in a:
        if torch.is_tensor(a[k]):
          assert torch.equal(a[k], b[k]), k
  # get_all gives every pixel's rays, and the selected ones at the sampled pixels
  ta, ra = outs[0][-1]
  ga = s.get_all(ta)
  sel = torch.as_tensor(ra["selected_inds"]).cuda()
  for k in ("ray_o", "ray_d", "uv_grid", "rgb"):
    assert torch.equal(ga[k][sel], ra[k]), k
  assert torch.equal(ga["flows"][:, sel], ra["flows"])


def test_training_step_from_scene_matches_host_path(tmp_path):
  from dynibar_b200 import criterion as cr, feature_network, mono_scene, render_ray as rr, sample_ray, synthetic
  from dynibar_b200.projection import Projector
  dev = torch.device("cuda:0")
  n, H, W = 16, 48, 64
  path = msr.write_scene(str(tmp_path / "s" / "dense"), msr.synthetic_scene(21, n, H, W, mask_hw=(40, 70)))
  sargs = SimpleNamespace(training_height=H, num_source_views=3, max_range=9, num_vv=3, mask_src_view=True,
                          erosion_radius=3, init_decay_epoch=150)
  scene = mono_scene.MonocularScene(path, sargs, dev)
  scene.set_epoch(0)
  sample_ray.rng = np.random.RandomState(3)
  td, rb = scene.sample(np.random.RandomState(4), 256, "center")
  sample_ray.rng = np.random.RandomState(3)
  host = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in td.items()}
  rb_host = sample_ray.RaySamplerSingleImage(host, dev).random_sample(256, "center")
  assert np.array_equal(rb_host["selected_inds"], rb["selected_inds"])

  args = synthetic.make_args(1, 1, 0)
  args = SimpleNamespace(**dict(vars(args), w_disp=5e-2, w_flow=5e-3, w_cycle=0.1, cycle_factor=0.1,
                                anneal_cycle=False, w_reg=0.05, w_skew_entropy=1e-3, w_distortion=1e-3,
                                decay_rate=10.0, init_decay_epoch=150))
  losses = []
  grads = []
  for batch in (rb, rb_host):
    model, args = synthetic.make_model(32, 0, num_frames=n, args=args, seed=3, mono=True)
    model = synthetic.model_to(model, dev)
    params = []
    for m in (model.net_coarse_dy, model.net_coarse_st, model.motion_mlp):
      m.requires_grad_(True)
      params += list(m.parameters())
    torch.manual_seed(5)
    enc = feature_network.ResNet().to(dev).requires_grad_(True)
    opt = torch.optim.Adam(params + list(enc.parameters()), lr=1e-4)
    i, a = int(td["id"]), int(td["anchor_id"])
    offs = ([int(j) - i for j in td["nearest_pose_ids"][0]], [int(j) - a for j in td["anchor_nearest_pose_ids"][0]])
    t = (td["ref_time"], td["anchor_time"])
    with rr.precision_scope("fp32"):
      fm = tuple(enc(batch[k][0].permute(0, 3, 1, 2).contiguous())[0]
                 for k in ("src_rgbs", "anchor_src_rgbs", "static_src_rgbs"))
      ret = rr.render_rays_mono((i, a), t, offs, batch, model, fm, Projector(dev), 32, args, inv_uniform=True,
                                det=True, is_train=True, num_vv=3)
      loss, _ = cr.mono_step_loss(ret, batch, args, 0)
      opt.zero_grad(set_to_none=True)
      loss.backward()
    g = [p.grad for p in params + list(enc.parameters()) if p.grad is not None]
    assert g and all(torch.isfinite(x).all() for x in g)
    opt.step()
    losses.append(loss.item())
    grads.append(len(g))
  print("loss from the scene %.9g, from the host path %.9g" % tuple(losses))
  assert abs(losses[0] - losses[1]) <= 1e-6 * abs(losses[1]), losses
  assert grads[0] == grads[1]
