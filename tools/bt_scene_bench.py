"""A monocular bullet-time sweep from files, two ways, on one GPU.

  python tools/bt_scene_bench.py [--cameras 50] [--frames 30] [--render-idx 15] [--reps 1]

A synthetic scene is written to a temporary `dense` folder (288x512 frames and virtual views as PNG, 1-channel
dynamic masks) and swept with render_monocular_bt.py's configuration (configs/test_kid-running.txt: 7 source views,
max_range 10, 3 virtual views, mask_src_view) at 64 samples, chunks of 8192 rays, with a randomly initialised
model.

  scene      BulletTimeScene: the scene is read once (timed on its own), then the sweep from the device-resident
             scene: per group of up to 16 cameras the pools and rays on the device, one encoder pass per pool, one
             render_multi_image_mono, the frame kernel and one copy of the uint8 frames.
  reference  the script's flow, camera by camera: a cv2 restatement of DynamicVideoDataset.__getitem__ (its ground
             truth, 7 temporal frames, 3 virtual views, 15 static frames and their masks, read from the PNGs),
             RaySamplerSingleImage.get_all, the encoder over the camera's 10 + 15 views, render_single_image_mono and
             the numpy uint8 conversion.

Both arms include the frames' trip to the host; neither writes PNGs.  Prints one JSON line: each arm's seconds per
sweep (host clock around device-synchronised work, best of the reps), the reference arm's loader share (the
__getitem__ restatement timed on its own), whether the two arms' frames are equal, and the GPU model, power limit and
SM clock the numbers were measured at.
"""

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def parse():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--cameras", type=int, default=50, help="cameras of the reference arm (the scene arm sweeps 50)")
  ap.add_argument("--frames", type=int, default=30)
  ap.add_argument("--render-idx", type=int, default=15)
  ap.add_argument("--H", type=int, default=288)
  ap.add_argument("--W", type=int, default=512)
  ap.add_argument("--samples", type=int, default=64)
  ap.add_argument("--chunk", type=int, default=8192)
  ap.add_argument("--reps", type=int, default=1, help="timed sweeps per arm (after one warm-up sweep each)")
  ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
  return ap.parse_args()


def gpu_info(index):
  name = torch.cuda.get_device_name(index)
  try:
    out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = "unknown"
  return {"name": name, "power_limit, sm_clock, max_sm_clock": out}


def write_scene(root, n, H, W, seed=0):
  """A synthetic monocular scene: LLFF poses drifting along x, 8 virtual views per frame, random frames / views /
  masks, as lossless PNGs."""
  import cv2

  def png(path, a):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    cv2.imwrite(path, np.ascontiguousarray(a[:, :, ::-1] if a.ndim == 3 else a))

  rng = np.random.RandomState(seed)
  poses = []
  for i in range(n):
    c = np.array([0.02 * i, rng.normal(0, 0.003), rng.normal(0, 0.003)])
    poses.append(np.concatenate([np.eye(3), c[:, None], np.array([[2 * H], [2 * W], [0.78 * W]])], 1))
  bds = np.stack([rng.uniform(1.0, 2.0, n), rng.uniform(4.0, 8.0, n)], 1)
  os.makedirs(root, exist_ok=True)
  np.save(os.path.join(root, "poses_bounds_cvd.npy"), np.concatenate([np.stack(poses).reshape(n, 15), bds], 1))
  vv = np.stack([[np.concatenate([np.eye(3), (p[:, 3] + rng.normal(0, 0.02, 3))[:, None]], 1) for _ in range(8)]
                 for p in poses])
  np.save(os.path.join(root, "source_vv_poses.npy"), np.ascontiguousarray(np.transpose(vv, (1, 2, 3, 0))))
  png(os.path.join(root, "images", "00000.png"), np.zeros((2 * H, 2 * W, 3), np.uint8))
  base = rng.randint(0, 256, (H, W, 3)).astype(np.uint8)
  for i in range(n):
    png(os.path.join(root, "images_%dx%d" % (W, H), "%05d.png" % i), np.roll(base, 3 * i, 1))
    m = np.full((H, W), 255, np.uint8)
    m[H // 3:H // 2, (5 * i) % W:(5 * i) % W + W // 8] = 0
    png(os.path.join(root, "dynamic_masks", "%d.png" % i), m)
    for j in range(8):
      png(os.path.join(root, "source_virtual_views_%dx%d" % (W, H), "%05d" % i, "%02d.png" % j),
                    np.roll(base, 3 * i + j, 0))


def main():
  a = parse()
  if not torch.cuda.is_available():
    raise SystemExit("bt_scene_bench: needs a GPU")
  import cv2
  from dynibar_b200 import render_ray as rr, sample_ray as sr, synthetic
  from dynibar_b200.bt_scene import BulletTimeScene, OFFSETS
  from dynibar_b200.feature_network import ResNet
  from dynibar_b200.projection import Projector
  from dynibar_b200.render_image import render_single_image_mono

  dev = torch.device("cuda", 0)
  rr.set_precision(a.precision)
  model, args = synthetic.make_model(a.samples, 0, num_frames=a.frames, mono=True)
  model = synthetic.model_to(model, dev)
  torch.manual_seed(1)
  model.feature_net = ResNet().to(dev).eval().requires_grad_(False)
  model.feature_net_st = ResNet().to(dev).eval().requires_grad_(False)
  args.anti_alias_pooling, args.mask_rgb = 1, 1
  vars(args).update(training_height=a.H, num_source_views=7, max_range=10, num_vv=3, mask_src_view=True,
                    render_idx=a.render_idx, N_samples=a.samples, N_importance=0, chunk_size=a.chunk,
                    inv_uniform=True, white_bkgd=False)
  P = Projector(dev)

  def sync_time():
    torch.cuda.synchronize(dev)
    return time.perf_counter()

  with tempfile.TemporaryDirectory() as tmp:
    root = os.path.join(tmp, "scene", "dense")
    write_scene(root, a.frames, a.H, a.W)
    t0 = sync_time()
    scene = BulletTimeScene(root, args, dev)
    load_s = sync_time() - t0
    plan, cams = scene.plan, scene.cams
    files = cams["rgb_files"]
    H, W = scene.H, scene.W

    def scene_sweep():
      return np.concatenate([f for _, f in scene.sweep(model, P, args)])

    def read_rgb(path):
      return cv2.imread(path)[:, :, ::-1].astype(np.float32) / 255.0

    def item(k):
      """DynamicVideoDataset.__getitem__ restated with cv2 (render_monocular_bt.py:96-259)."""
      t, vv, st = plan["selections"][k]
      read_rgb(files[min(k, len(files) - 1)])  # the unused ground truth
      src = [read_rgb(files[f]) for f in t]
      src_cams = [scene._cam_rows[f] for f in t]
      vdir = os.path.join(root, "source_virtual_views_%dx%d" % (W, H), "%05d" % a.render_idx)
      for j in vv:
        src.append(read_rgb(os.path.join(vdir, "%02d.png" % j)))
        src_cams.append(np.concatenate(([H, W], plan["render_K"][k].reshape(-1),
                                        cams["vv_c2w"][a.render_idx, j].reshape(-1))).astype(np.float32))
      static = []
      for f in st:
        m = cv2.imread(os.path.join(root, "dynamic_masks", "%d.png" % f), cv2.IMREAD_UNCHANGED)
        m = cv2.resize(m.astype(np.float32) / 255.0, (W, H), interpolation=cv2.INTER_NEAREST)
        static.append(read_rgb(files[f]) * (m[..., None] if m.ndim == 2 else m))
      return dict(camera=torch.from_numpy(plan["cameras"][k])[None],
                  depth_range=torch.from_numpy(scene.depth_range)[None],
                  src_rgbs=torch.from_numpy(np.stack(src))[None], src_cameras=torch.from_numpy(np.stack(src_cams))[None],
                  static_src_rgbs=torch.from_numpy(np.stack(static))[None],
                  static_src_cameras=torch.from_numpy(scene._cam_rows[st])[None])

    ref_time = torch.tensor([a.render_idx / float(a.frames)], dtype=torch.float64, device=dev)

    def reference_sweep():
      out = []
      for k in range(a.cameras):
        smp = sr.RaySamplerSingleImage(item(k), dev)
        rb = smp.get_all()
        with torch.no_grad():
          ref = model.feature_net(rb["src_rgbs"].squeeze(0).permute(0, 3, 1, 2))[0]
          st = model.feature_net_st(rb["static_src_rgbs"].squeeze(0).permute(0, 3, 1, 2))[0]
          ret = render_single_image_mono((a.render_idx, None), (ref_time, None), (list(OFFSETS), None), smp, rb,
                                         model, P, a.chunk, a.samples, args, inv_uniform=True, det=True,
                                         featmaps=(ref, None, st), is_train=False, num_vv=3)
        x = ret["outputs_coarse_ref"]["rgb"].cpu().numpy()
        ch, cw = int(H * 0.03), int(W * 0.03)
        out.append((255 * np.clip(x, a_min=0, a_max=1.0)).astype(np.uint8)[ch:H - ch, cw:W - cw])
      return np.stack(out)

    def loader_only():
      for k in range(a.cameras):
        item(k)

    def timed(fn):
      t0 = sync_time()
      out = fn()
      return sync_time() - t0, out

    for fn in (scene_sweep, reference_sweep):  # warm-up
      timed(fn)
    t_scene, t_ref, t_load = [], [], []
    for _ in range(a.reps):
      dt, f_scene = timed(scene_sweep)
      t_scene.append(dt)
      dt, f_ref = timed(reference_sweep)
      t_ref.append(dt)
      t_load.append(timed(loader_only)[0])
    same = np.array_equal(f_scene[:a.cameras], f_ref)
    diff = int(np.abs(f_scene[:a.cameras].astype(np.int32) - f_ref.astype(np.int32)).max())
    print(json.dumps({
        "what": "bullet-time sweep from files: %d frames at %dx%d, 7+3 dynamic / 15 static views, mask_src_view, %d "
                "samples, chunk %d, %s" % (a.frames, a.W, a.H, a.samples, a.chunk, a.precision),
        "groups": [hi - lo for lo, hi in scene.groups], "scene_load_s": load_s, "scene_mb": scene.nbytes / 1e6,
        "scene_sweep_s_50_cameras": min(t_scene), "scene_all_reps_s": t_scene,
        "reference_cameras": a.cameras, "reference_sweep_s": min(t_ref), "reference_all_reps_s": t_ref,
        "reference_loader_s": min(t_load), "reference_loader_share": min(t_load) / min(t_ref),
        "speedup_per_camera": (min(t_ref) / a.cameras) / (min(t_scene) / 50),
        "frames_equal": bool(same), "frames_max_abs_diff": diff,
        "timing": "host clock around device-synchronised work, best of the reps, after one warm-up of each arm",
        "gpu": gpu_info(dev.index),
    }))


if __name__ == "__main__":
  main()
