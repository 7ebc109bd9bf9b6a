"""The bullet-time scene on the GPU against the reference's render_monocular_bt.py loader (tests/golden/bt_scene.pt):
every camera's pooled views bit-equal to the fixture's (by SHA-256), each group's device-built batch equal to
stack_pooled_ray_batches of the per-camera get_all() batches, the uint8 frames bit-identical to the renderer's output
converted as the script does, no host synchronisation while a group is assembled, the tool's PNGs, and the
refusals."""

import os
import shutil
import types

import cv2
import numpy as np
import pytest
import torch

import bt_scene_ref as bsr
from dynibar_b200 import bt_scene, sample_ray as sr, synthetic
from dynibar_b200.feature_network import ResNet
from dynibar_b200.projection import Projector

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bt_scene.pt")
DEV = torch.device("cuda", 0)
N_SAMPLES = 16


@pytest.fixture(scope="module")
def golden():
  return bsr.load_golden(GOLDEN)


@pytest.fixture(scope="module")
def roots(golden, tmp_path_factory):
  base = tmp_path_factory.mktemp("bt")
  return {name: bsr.write_scene(str(base / name / "dense"), s) for name, s in golden["scenes"].items()}


def _args(case, **kw):
  a = dict(training_height=bsr.SCENE_H, num_source_views=case["num_source_views"], max_range=case["max_range"],
           num_vv=case["num_vv"], mask_src_view=case["mask_src_view"], render_idx=case["render_idx"],
           N_samples=N_SAMPLES, N_importance=0, chunk_size=2048, inv_uniform=True, white_bkgd=False,
           anti_alias_pooling=1, mask_rgb=1, occ_weights_mode=0, num_basis=6, input_dir=True, input_xyz=False,
           coarse_feat_dim=32, fine_feat_dim=32)
  a.update(kw)
  return types.SimpleNamespace(**a)


def _host_views(scene, case, k):
  """Camera k's source images as the reference builds them (float32 u8 / 255, the static ones times the
  nearest-resized raw mask / 255); test_bt_scene_host_cpu shows this equals the fixture's images."""
  t, vv, st = case["selections"][k]
  src = [scene["frames"][f] for f in t] + [scene["vviews"][case["render_idx"]][j] for j in vv]
  src = np.stack(src).astype(np.float32) / 255.0
  out = []
  for f in st:
    rgb = scene["frames"][f].astype(np.float32) / 255.0
    if case["mask_src_view"]:
      m = cv2.resize(scene["masks"][f].astype(np.float32) / 255.0, (bsr.SCENE_W, bsr.SCENE_H),
                     interpolation=cv2.INTER_NEAREST)
      rgb = rgb * (m[..., None] if m.ndim == 2 else m)
    out.append(rgb)
  return torch.from_numpy(src), torch.from_numpy(np.stack(out))


def _host_group(golden, case, lo, hi):
  scene = golden["scenes"][case["scene"]]
  batches, dy, st = [], [], []
  for k in range(lo, hi):
    s, t = _host_views(scene, case, k)
    batches.append(bsr.item_batch(case, k, s, t, DEV))
    d, s_ = bsr.ids_of(case, k)
    dy.append(d)
    st.append(s_)
  return sr.stack_pooled_ray_batches(batches, dy, st)[0]


def test_pools_equal_fixture_images_and_batches_equal_pooled_batches(golden, roots):
  seen_images = 0
  for case in golden["cases"]:
    scene = bt_scene.BulletTimeScene(roots[case["scene"]], _args(case), DEV)
    assert scene.nbytes > 0 and len(scene) == len(scene.groups)
    for g, (lo, hi) in enumerate(scene.groups):
      step = scene.group_batch(g)
      rb = step["ray_batch"]
      assert step["cameras"] == list(range(lo, hi)) and step["frame_idx"] == (case["render_idx"], None)
      assert step["time_offset"] == ([-3, -2, -1, 0, 1, 2, 3], None)
      assert step["time_embedding"][0].dtype == torch.float64
      assert step["time_embedding"][0].item() == float(case["render_idx"] / float(bsr.N_FRAMES))
      for k, (src, st) in case["images"].items():
        if lo <= k < hi:
          seen_images += 1
          assert bsr.digest(rb["src_rgbs"][0][rb["src_views"][k - lo].long()]) == src
          assert bsr.digest(rb["static_src_rgbs"][0][rb["static_src_views"][k - lo].long()]) == st
      want = _host_group(golden, case, lo, hi)
      assert sorted(k for k in want if want[k] is not None) == sorted(k for k in rb if rb[k] is not None)
      for key, w in want.items():
        got = rb[key]
        if key == "ray_d":  # a different float32 summation order than torch's CPU matmul (DESIGN §3.8)
          assert (got - w).abs().max().item() <= 2.4e-7, key
        elif torch.is_tensor(w):
          assert got.dtype == w.dtype and got.shape == w.shape and got.device.type == w.device.type, key
          assert torch.equal(got, w), key
        else:
          assert got == w, key
  assert seen_images == 50 * len(golden["cases"])


def _model(seed=2):
  model, args = synthetic.make_model(N_SAMPLES, 0, num_frames=bsr.N_FRAMES, mono=True, seed=seed)
  model = synthetic.model_to(model, DEV)
  torch.manual_seed(seed)
  model.feature_net = ResNet().to(DEV).eval().requires_grad_(False)
  model.feature_net_st = ResNet().to(DEV).eval().requires_grad_(False)
  return model


def _numpy_frames(rgb):
  x = rgb.cpu().numpy()
  h, w = x.shape[1:3]
  ch, cw = int(h * 0.03), int(w * 0.03)
  return (255 * np.clip(x, a_min=0, a_max=1.0)).astype(np.uint8)[:, ch:h - ch, cw:w - cw]


def test_sweep_frames_equal_host_batch_render(golden, roots):
  from dynibar_b200.render_image import render_multi_image_mono
  model, P = _model(), Projector(DEV)
  for case in (golden["cases"][0], golden["cases"][2]):  # 1- and 3-channel masks, both ends of the video
    args = _args(case)
    scene = bt_scene.BulletTimeScene(roots[case["scene"]], args, DEV)
    swept = list(scene.sweep(model, P, args))
    assert [c for cams, _ in swept for c in cams] == list(range(50))
    for g, (lo, hi) in enumerate(scene.groups):
      cams, frames = swept[g]
      assert frames.dtype == np.uint8 and frames.shape == (hi - lo, bsr.SCENE_H - 2, bsr.SCENE_W - 2, 3)
      step = scene.group_batch(g)
      host = _host_group(golden, case, lo, hi)
      host["ray_d"] = step["ray_batch"]["ray_d"]  # the rays agree within 2.4e-7 (above); render on the same rays
      with torch.no_grad():
        ref = model.feature_net(host["src_rgbs"].squeeze(0).permute(0, 3, 1, 2))[0]
        st = model.feature_net_st(host["static_src_rgbs"].squeeze(0).permute(0, 3, 1, 2))[0]
        rets = render_multi_image_mono((case["render_idx"], None), step["time_embedding"], step["time_offset"],
                                       step["ray_samplers"], host, model, P, args.chunk_size, N_SAMPLES, args,
                                       inv_uniform=True, det=True, featmaps=(ref, None, st), is_train=False,
                                       num_vv=args.num_vv)
      rgb = torch.stack([r["outputs_coarse_ref"]["rgb"] for r in rets])
      np.testing.assert_array_equal(frames, _numpy_frames(rgb))


def test_frame_conversion_matches_numpy():
  g = torch.Generator().manual_seed(0)
  K, H, W = 3, 100, 201  # crop 3 x 6
  x = torch.rand(K, H, W, 3, generator=g) * 1.4 - 0.2
  steps = torch.arange(256, dtype=torch.float32) / 255.0
  special = torch.cat([torch.tensor([0.0, -0.0, 1.0, -1e-30, 1e-30, 1.0 + 1e-7, 2.0, -3.0, float("inf"),
                                     float("-inf")]),
                       steps, torch.nextafter(steps, torch.zeros(())), torch.nextafter(steps, torch.ones(()))])
  x.view(-1)[:special.numel()] = special  # partly in the cropped-off border
  inner = x[1, 5:7, 6:W - 6].clone().reshape(-1)
  inner[:special.numel()] = special
  x[1, 5:7, 6:W - 6] = inner.reshape(2, W - 12, 3)  # and inside the window
  got = bt_scene.bt_frames(x.to(DEV)).cpu().numpy()
  assert got.shape == (K, H - 6, W - 12, 3)
  np.testing.assert_array_equal(got, _numpy_frames(x))


def test_group_assembly_and_frames_do_not_synchronise(golden, roots):
  case = golden["cases"][2]
  scene = bt_scene.BulletTimeScene(roots[case["scene"]], _args(case), DEV)
  rgb = torch.rand(16, bsr.SCENE_H, bsr.SCENE_W, 3, device=DEV)
  a = [scene.group_batch(g) for g in range(len(scene))]
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode("error")
  try:
    # twice over the sweep: more groups than staging buffers
    b = [scene.group_batch(g) for g in range(len(scene))] + [scene.group_batch(g) for g in range(len(scene))]
    f = scene.frames_device(rgb[:a[0]["ray_batch"]["camera"].shape[0]])
  finally:
    torch.cuda.set_sync_debug_mode(0)
  assert f.dtype == torch.uint8
  for x, y in zip(a + a, b):
    for k, v in x["ray_batch"].items():
      if torch.is_tensor(v):
        assert torch.equal(v, y["ray_batch"][k]), k


def test_tool_writes_the_sweep(golden, roots, tmp_path):
  import sys
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
  import render_monocular_bt as tool
  from dynibar_b200 import model as dm
  case = golden["cases"][0]
  model = _model(seed=4)
  enc = {k: getattr(model, k).state_dict() for k in ("feature_net", "feature_net_st")}
  coarse, _ = dm.checkpoint_dicts(model, global_step=1234, encoders=enc)
  ckpt = str(tmp_path / "model.pth")
  torch.save(coarse, ckpt)
  argv = ["--scene_path", roots["A"], "--coarse", ckpt, "--render_idx", str(case["render_idx"]), "--out",
          str(tmp_path / "out"), "--training_height", str(bsr.SCENE_H), "--num_source_views",
          str(case["num_source_views"]), "--max_range", str(case["max_range"]), "--num_vv", str(case["num_vv"]),
          "--mask_src_view", "--N_samples", str(N_SAMPLES), "--chunk_size", "2048", "--inv_uniform"]
  out_dir = tool.main(argv)
  assert out_dir.endswith(os.path.join("exp", str(case["render_idx"]), "A_001234", "videos"))
  args = _args(case)
  loaded, info = dm.model_from_checkpoints(args, coarse=ckpt, mono=True, device=DEV)
  for k in ("feature_net", "feature_net_st"):
    e = ResNet().to(DEV)
    e.load_state_dict(dm._strip(info["encoders"][k]))
    setattr(loaded, k, e.eval().requires_grad_(False))
  scene = bt_scene.BulletTimeScene(roots["A"], args, DEV)
  frames = np.concatenate([f for _, f in scene.sweep(loaded, Projector(DEV), args)])
  assert sorted(os.listdir(os.path.join(out_dir, "rgb_out"))) == sorted("%d.png" % i for i in range(50))
  for i in range(50):
    png = cv2.imread(os.path.join(out_dir, "rgb_out", "%d.png" % i))[:, :, ::-1]
    np.testing.assert_array_equal(png, frames[i])


def test_errors(golden, roots, tmp_path):
  case = golden["cases"][0]
  with pytest.raises(ValueError, match="render_idx"):
    bt_scene.BulletTimeScene(roots["A"], _args(case, render_idx=2), DEV)
  with pytest.raises(ValueError, match="render_idx"):
    bt_scene.BulletTimeScene(roots["A"], _args(case, render_idx=bsr.N_FRAMES - 3), DEV)
  bt_scene.BulletTimeScene(roots["B"], _args(case, render_idx=bsr.N_FRAMES - 4), DEV)  # scene B holds frame 12's views

  def broken(name, fn):
    root = str(tmp_path / name / "dense")
    shutil.copytree(roots["A"], root)
    fn(root)
    return root

  W, H = bsr.SCENE_W, bsr.SCENE_H
  no_vv = broken("novv", lambda r: shutil.rmtree(os.path.join(r, "source_virtual_views_%dx%d" % (W, H), "00003")))
  with pytest.raises(ValueError, match="missing directory"):
    bt_scene.BulletTimeScene(no_vv, _args(case), DEV)
  no_masks = broken("nomasks", lambda r: shutil.rmtree(os.path.join(r, "dynamic_masks")))
  with pytest.raises(ValueError, match="missing directory"):
    bt_scene.BulletTimeScene(no_masks, _args(case), DEV)
  bt_scene.BulletTimeScene(no_masks, _args(case, mask_src_view=False), DEV)  # masks are read only when asked
  few = broken("few", lambda r: os.remove(os.path.join(r, "dynamic_masks", "15.png")))
  with pytest.raises(ValueError, match="15 dynamic masks"):
    bt_scene.BulletTimeScene(few, _args(case), DEV)
  big = broken("big", lambda r: bsr.write_png(os.path.join(r, "images_%dx%d" % (W, H), "00005.png"),
                                              np.zeros((H, W + 2, 3), np.uint8)))
  with pytest.raises(ValueError, match="frame"):
    bt_scene.BulletTimeScene(big, _args(case), DEV)
  vv_big = broken("vvbig", lambda r: bsr.write_png(
      os.path.join(r, "source_virtual_views_%dx%d" % (W, H), "00003", "02.png"), np.zeros((H + 1, W, 3), np.uint8)))
  with pytest.raises(ValueError, match="virtual view"):
    bt_scene.BulletTimeScene(vv_big, _args(case), DEV)
  with pytest.raises(ValueError, match="num_vv"):
    bt_scene.BulletTimeScene(roots["A"], _args(case, num_vv=9), DEV)
