"""The stabilised video (render_idx < 0) on the GPU against the reference's render_monocular_bt.py loader
(tests/golden/bt_stab.pt): every camera's pools hash to the fixture's digests, each group's device-built batch equals
the host-built get_all() batch of the camera's item, the frames are bit-identical to render_single_image_mono on that
batch converted as the script does, no host synchronisation while a group is assembled, the tool's PNGs, and the
errors."""

import os
import shutil
import sys
import types

import cv2
import numpy as np
import pytest
import torch

import bt_scene_ref as bsr
import bt_stab_ref as bst
from dynibar_b200 import bt_scene, sample_ray as sr, synthetic
from dynibar_b200.feature_network import ResNet
from dynibar_b200.projection import Projector

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bt_stab.pt")
DEV = torch.device("cuda", 0)
N_SAMPLES = 16
RENDERED = list(range(bst.FIRST, bst.LAST + 1))


@pytest.fixture(scope="module")
def golden():
  return bst.load_golden(GOLDEN)


@pytest.fixture(scope="module")
def roots(golden, tmp_path_factory):
  base = tmp_path_factory.mktemp("stab")
  return {name: bsr.write_scene(str(base / name / "dense"), s) for name, s in golden["scenes"].items()}


def _args(case, **kw):
  a = dict(training_height=bsr.SCENE_H, num_source_views=case["num_source_views"], max_range=case["max_range"],
           num_vv=case["num_vv"], mask_src_view=case["mask_src_view"], render_idx=-1, N_samples=N_SAMPLES,
           N_importance=0, chunk_size=2048, inv_uniform=True, white_bkgd=False, anti_alias_pooling=1, mask_rgb=1,
           occ_weights_mode=0, num_basis=6, input_dir=True, input_xyz=False, coarse_feat_dim=32, fine_feat_dim=32)
  a.update(kw)
  return types.SimpleNamespace(**a)


def _host_item(scene, case, i):
  """Camera i's item as the reference builds it: the source images (float32 u8 / 255: temporal frames, frame i's
  virtual views, static frames times the nearest-resized raw mask / 255) with the fixture's cameras."""
  k = i - bst.FIRST
  t, vv, st = case["selections"][k]
  src = np.stack([scene["frames"][f] for f in t] + [scene["vviews"][i][j] for j in vv]).astype(np.float32) / 255.0
  static = []
  for f in st:
    rgb = scene["frames"][f].astype(np.float32) / 255.0
    if case["mask_src_view"]:
      m = cv2.resize(scene["masks"][f].astype(np.float32) / 255.0, (bsr.SCENE_W, bsr.SCENE_H),
                     interpolation=cv2.INTER_NEAREST)
      rgb = rgb * (m[..., None] if m.ndim == 2 else m)
    static.append(rgb)
  return dict(camera=case["camera"][k][None], depth_range=case["depth_range"][None],
              src_rgbs=torch.from_numpy(src)[None], src_cameras=case["src_cameras"][k][None],
              static_src_rgbs=torch.from_numpy(np.stack(static))[None],
              static_src_cameras=case["static_src_cameras"][k][None])


def _host_pooled(golden, case, i):
  """stack_pooled_ray_batches of camera i's get_all() batch, the pools named as the stabilised plan names them."""
  batch = sr.RaySamplerSingleImage(_host_item(golden["scenes"][case["scene"]], case, i), DEV).get_all()
  t, vv, st = case["selections"][i - bst.FIRST]
  return sr.stack_pooled_ray_batches([batch], [list(t) + [("vv", i, j) for j in vv]], [list(st)])[0]


def test_pools_and_batches_equal_reference_items(golden, roots):
  for case in golden["cases"]:
    scene = bt_scene.BulletTimeScene(roots[case["scene"]], _args(case), DEV)
    assert scene.stabilized and scene.groups == [(i, i + 1) for i in RENDERED]
    assert scene.nbytes >= bsr.N_FRAMES * 9 * bsr.SCENE_H * bsr.SCENE_W * 3  # every frame's 8 virtual views
    for g, i in enumerate(RENDERED):
      k = i - bst.FIRST
      step = scene.group_batch(g)
      rb = step["ray_batch"]
      assert step["cameras"] == [i] and step["frame_idx"] == (i, None)
      assert step["time_offset"] == ([-3, -2, -1, 0, 1, 2, 3], None)
      te = step["time_embedding"][0]
      assert te.dtype == torch.float64 and te.shape == (1,) and te.item() == case["ref_time"][k]
      src, st = case["images"][i]
      assert bsr.digest(rb["src_rgbs"][0][rb["src_views"][0].long()]) == src
      assert bsr.digest(rb["static_src_rgbs"][0][rb["static_src_views"][0].long()]) == st
      want = _host_pooled(golden, case, i)
      assert sorted(x for x in want if want[x] is not None) == sorted(x for x in rb if rb[x] is not None)
      for key, w in want.items():
        got = rb[key]
        if key == "ray_d":  # a different float32 summation order than torch's matmul (DESIGN §3.8)
          assert (got - w).abs().max().item() <= 2.4e-7, key
        elif torch.is_tensor(w):
          assert got.dtype == w.dtype and got.shape == w.shape and got.device.type == w.device.type, key
          assert torch.equal(got, w), key
        else:
          assert got == w, key


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


def test_video_frames_equal_single_image_render(golden, roots):
  from dynibar_b200.render_image import render_single_image_mono
  model, P = _model(), Projector(DEV)
  for case in golden["cases"]:  # masked 3-channel static views with 3 virtual views; unmasked with 2
    args = _args(case)
    scene = bt_scene.BulletTimeScene(roots[case["scene"]], args, DEV)
    swept = list(scene.sweep(model, P, args))
    assert [c for cams, _ in swept for c in cams] == RENDERED
    for g, i in enumerate(RENDERED):
      cams, frames = swept[g]
      assert frames.dtype == np.uint8 and frames.shape == (1, bsr.SCENE_H - 2, bsr.SCENE_W - 2, 3)
      step = scene.group_batch(g)
      smp = sr.RaySamplerSingleImage(_host_item(golden["scenes"][case["scene"]], case, i), DEV)
      rb = smp.get_all()
      rb["ray_d"] = step["ray_batch"]["ray_d"]  # the rays agree within 2.4e-7 (above); render on the same rays
      ref_time = torch.tensor([case["ref_time"][i - bst.FIRST]], dtype=torch.float64, device=DEV)
      offsets = [f - i for f in case["selections"][i - bst.FIRST][0]]
      with torch.no_grad():
        ref = model.feature_net(rb["src_rgbs"].squeeze(0).permute(0, 3, 1, 2))[0]
        st = model.feature_net_st(rb["static_src_rgbs"].squeeze(0).permute(0, 3, 1, 2))[0]
        ret = render_single_image_mono((i, None), (ref_time, None), (offsets, None), smp, rb, model, P,
                                       args.chunk_size, N_SAMPLES, args, inv_uniform=True, det=True,
                                       featmaps=(ref, None, st), is_train=False, num_vv=args.num_vv)
      np.testing.assert_array_equal(frames, _numpy_frames(ret["outputs_coarse_ref"]["rgb"][None]))


def test_group_assembly_does_not_synchronise(golden, roots):
  case = golden["cases"][0]
  scene = bt_scene.BulletTimeScene(roots[case["scene"]], _args(case), DEV)
  rgb = torch.rand(1, bsr.SCENE_H, bsr.SCENE_W, 3, device=DEV)
  a = [scene.group_batch(g) for g in range(len(scene))]
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode("error")
  try:
    # twice over the video: more groups than staging buffers
    b = [scene.group_batch(g) for g in range(len(scene))] + [scene.group_batch(g) for g in range(len(scene))]
    f = scene.frames_device(rgb)
  finally:
    torch.cuda.set_sync_debug_mode(0)
  assert f.dtype == torch.uint8
  for x, y in zip(a + a, b):
    assert x["frame_idx"] == y["frame_idx"]
    for k, v in x["ray_batch"].items():
      if torch.is_tensor(v):
        assert torch.equal(v, y["ray_batch"][k]), k


def test_tool_writes_the_video(golden, roots, tmp_path):
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
  import render_monocular_bt as tool
  from dynibar_b200 import model as dm
  case = golden["cases"][0]
  model = _model(seed=4)
  enc = {k: getattr(model, k).state_dict() for k in ("feature_net", "feature_net_st")}
  coarse, _ = dm.checkpoint_dicts(model, global_step=1234, encoders=enc)
  ckpt = str(tmp_path / "model.pth")
  torch.save(coarse, ckpt)
  argv = ["--scene_path", roots[case["scene"]], "--coarse", ckpt, "--render_idx", "-1", "--out",
          str(tmp_path / "out"), "--training_height", str(bsr.SCENE_H), "--num_source_views",
          str(case["num_source_views"]), "--max_range", str(case["max_range"]), "--num_vv", str(case["num_vv"]),
          "--mask_src_view", "--N_samples", str(N_SAMPLES), "--chunk_size", "2048", "--inv_uniform"]
  out_dir = tool.main(argv)
  assert out_dir.endswith(os.path.join("exp", "-1", "%s_001234" % case["scene"], "videos"))
  args = _args(case)
  loaded, info = dm.model_from_checkpoints(args, coarse=ckpt, mono=True, device=DEV)
  for k in ("feature_net", "feature_net_st"):
    e = ResNet().to(DEV)
    e.load_state_dict(dm._strip(info["encoders"][k]))
    setattr(loaded, k, e.eval().requires_grad_(False))
  scene = bt_scene.BulletTimeScene(roots[case["scene"]], args, DEV)
  swept = [(c, f) for cams, frames in scene.sweep(loaded, Projector(DEV), args) for c, f in zip(cams, frames)]
  names = os.listdir(os.path.join(out_dir, "rgb_out"))
  assert len(names) == bsr.N_FRAMES - 6 and sorted(names) == sorted("%d.png" % i for i in RENDERED)
  assert [c for c, _ in swept] == RENDERED
  for i, frame in swept:
    png = cv2.imread(os.path.join(out_dir, "rgb_out", "%d.png" % i))[:, :, ::-1]
    np.testing.assert_array_equal(png, frame)


def test_errors(golden, roots, tmp_path):
  case = golden["cases"][0]
  name = case["scene"]
  for r in (2, bsr.N_FRAMES - 3):  # the bullet-time sweep's bounds are unchanged
    with pytest.raises(ValueError, match="render_idx"):
      bt_scene.BulletTimeScene(roots[name], _args(case, render_idx=r), DEV)
  bt_scene.BulletTimeScene(roots[name], _args(case, render_idx=-2), DEV)  # any negative index: the video

  W, H = bsr.SCENE_W, bsr.SCENE_H
  for f in (0, bsr.N_FRAMES - 1):  # every frame's virtual views are read, rendered camera or not
    root = str(tmp_path / ("novv%d" % f) / "dense")
    shutil.copytree(roots[name], root)
    shutil.rmtree(os.path.join(root, "source_virtual_views_%dx%d" % (W, H), "%05d" % f))
    with pytest.raises(ValueError, match="missing directory .*%05d" % f):
      bt_scene.BulletTimeScene(root, _args(case), DEV)
  with pytest.raises(ValueError, match="num_vv"):
    bt_scene.BulletTimeScene(roots[name], _args(case, num_vv=9), DEV)

  s = golden["scenes"][name]
  short = dict(s, poses_bounds=s["poses_bounds"][:6], vv_poses=s["vv_poses"][..., :6], frames=s["frames"][:6],
               vviews={f: s["vviews"][f] for f in range(6)}, masks=s["masks"][:6])
  root = bsr.write_scene(str(tmp_path / "short" / "dense"), short)
  with pytest.raises(ValueError, match="at least 7 frames"):
    bt_scene.BulletTimeScene(root, _args(case), DEV)
