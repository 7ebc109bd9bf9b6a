"""A monocular bullet-time sweep, rendered two ways, on one GPU.

  python tools/bullet_time_bench.py [--cameras 50] [--reps 2]

A synthetic video and the 50 target cameras of render_wander_path around one time step (render_monocular_bt.py),
each camera with its own source views as bullet_time.select_source_views picks them: 7 temporal + 3 virtual
dynamic views and 15 static views (configs/test_kid-running.txt: num_source_views 7, max_range 10, num_vv 3), at
512x288, 64 samples, chunks of 8192 rays.

  per-camera  the reference script's loop: per camera, the encoder over its 10 + 15 source images and
              render_single_image_mono;
  batched     bullet_time.group_cameras splits the sweep into groups of at most 16 cameras (pools of at most 32
              views); per group, the encoder over each pool once and render_multi_image_mono.

The two arms alternate.  Prints one JSON line: rays/s of each arm (all cameras' rays over the wall time of the
sweep, device-synchronised, best of the reps), the encoder's share of each (the encoder passes of one sweep timed
on their own), the largest difference between the two arms' images, and the GPU model and power limit the numbers
were measured on.
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def parse():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--cameras", type=int, default=50)
  ap.add_argument("--H", type=int, default=288)
  ap.add_argument("--W", type=int, default=512)
  ap.add_argument("--frames", type=int, default=40)
  ap.add_argument("--render-idx", type=int, default=20)
  ap.add_argument("--samples", type=int, default=64)
  ap.add_argument("--chunk", type=int, default=8192)
  ap.add_argument("--reps", type=int, default=2, help="timed sweeps per arm (after one warm-up sweep each)")
  ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
  return ap.parse_args()


def gpu_info(index):
  name = torch.cuda.get_device_name(index)
  try:
    out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = "unknown"
  return {"name": name, "power_limit": out}


def main():
  a = parse()
  if not torch.cuda.is_available():
    raise SystemExit("bullet_time_bench: needs a GPU")
  from dynibar_b200 import bullet_time as bt, render_ray as rr, sample_ray as sr, synthetic
  from dynibar_b200.feature_network import ResNet
  from dynibar_b200.projection import Projector
  from dynibar_b200.render_image import render_multi_image_mono, render_single_image_mono

  dev = torch.device("cuda", 0)
  rr.set_precision(a.precision)
  H, W, n_vv, nsv, max_range = a.H, a.W, 3, 7, 10
  rng = np.random.RandomState(5)

  # ---- a synthetic video: camera centres drifting along x, 8 virtual views per frame; the wander path ----
  def c2w_at(c):
    m = np.eye(4)
    m[:3, 3] = c
    return m

  train = np.stack([c2w_at([0.01 * (i - a.render_idx), rng.normal(0, 0.003), rng.normal(0, 0.003)])
                    for i in range(a.frames)])
  vv = np.stack([[c2w_at(train[i, :3, 3] + rng.normal(0, 0.02, 3)) for _ in range(8)] for i in range(a.frames)])
  f = 0.78 * W
  llff = np.concatenate([np.eye(3), train[a.render_idx, :3, 3:4], np.array([[H], [W], [f]])], 1)
  path = [np.concatenate([p[:, :4], [[0, 0, 0, 1]]], 0) for p in bt.wander_path(llff)][:a.cameras]
  sel = [bt.select_source_views(p, train, vv, a.render_idx, nsv, max_range, n_vv) for p in path]
  groups = bt.group_cameras(sel)

  batch, _, _, frame, t, _ = synthetic.make_scene(H=H, W=W, V_dy=1, V_st=1, rays=1, num_frames=a.frames,
                                                  frame_idx=a.render_idx)
  offs = ([-3, -2, -1, 0, 1, 2, 3], None)
  Kmat = sr.parse_camera(batch["camera"])[2][0]
  g = torch.Generator().manual_seed(7)
  images = {("f", i): torch.rand(H, W, 3, generator=g) for i in range(a.frames)}
  images.update({("vv", j): torch.rand(H, W, 3, generator=g) for j in range(8)})
  images = {k: v.to(dev) for k, v in images.items()}
  cam = lambda m: synthetic.camera_vector(H, W, Kmat, torch.from_numpy(m).float())

  def dy_ids(s):
    return list(s[0]) + [("vv", j) for j in s[1]]

  def view_batch(k):
    smp = sr.RaySamplerSingleImage(dict(depth_range=batch["depth_range"], camera=cam(path[k])[None]), dev)
    b = smp.get_all()
    di, si = dy_ids(sel[k]), sel[k][2]
    b["src_rgbs"] = torch.stack([images[("f", i) if not isinstance(i, tuple) else i] for i in di])[None]
    b["src_cameras"] = torch.stack([cam(train[i]) if not isinstance(i, tuple) else cam(vv[a.render_idx, i[1]])
                                    for i in di])[None].to(dev)
    b["static_src_rgbs"] = torch.stack([images[("f", i)] for i in si])[None]
    b["static_src_cameras"] = torch.stack([cam(train[i]) for i in si])[None].to(dev)
    return smp, b

  model, args = synthetic.make_model(a.samples, 0, num_frames=a.frames, mono=True)
  args.anti_alias_pooling, args.mask_rgb = 1, 1
  model = synthetic.model_to(model, dev)
  torch.manual_seed(1)
  model.feature_net = ResNet().to(dev).requires_grad_(False)
  P = Projector(dev)
  views = [view_batch(k) for k in range(len(path))]

  def encode(rb):
    """render_monocular_bt.py: the encoder over the dynamic and the static source images."""
    cb, _ = model.feature_net(rb["src_rgbs"].squeeze(0).permute(0, 3, 1, 2))
    _, st = model.feature_net(rb["static_src_rgbs"].squeeze(0).permute(0, 3, 1, 2))
    return cb, None, st

  pooled = []
  for lo, hi in groups:
    pb, _, _ = sr.stack_pooled_ray_batches([views[k][1] for k in range(lo, hi)], [dy_ids(s) for s in sel[lo:hi]],
                                           [s[2] for s in sel[lo:hi]])
    pooled.append(([views[k][0] for k in range(lo, hi)], pb))

  def px(r):
    r = r["outputs_coarse_ref"]
    return torch.cat([r["rgb"].reshape(-1, 3), r["depth"].reshape(-1, 1)], 1)

  def per_camera():
    out = []
    for smp, b in views:
      out.append(px(render_single_image_mono(frame, t, offs, smp, b, model, P, a.chunk, a.samples, args,
                                             inv_uniform=True, det=True, featmaps=encode(b), is_train=False,
                                             num_vv=n_vv)))
    return out

  def batched():
    out = []
    for smps, pb in pooled:
      rets = render_multi_image_mono(frame, t, offs, smps, pb, model, P, a.chunk, a.samples, args, inv_uniform=True,
                                     det=True, featmaps=encode(pb), is_train=False, num_vv=n_vv)
      out += [px(r) for r in rets]
    return out

  def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out

  enc_pc = lambda: [encode(b) for _, b in views]
  enc_b = lambda: [encode(pb) for _, pb in pooled]
  for fn in (per_camera, batched, enc_pc, enc_b):  # warm-up of every shape
    timed(fn)
  t_pc, t_b, e_pc, e_b = [], [], [], []
  for _ in range(a.reps):
    dt, px_pc = timed(per_camera)
    t_pc.append(dt)
    dt, px_b = timed(batched)
    t_b.append(dt)
    e_pc.append(timed(enc_pc)[0])
    e_b.append(timed(enc_b)[0])
  d = max((x - y).abs().max().item() for x, y in zip(px_pc, px_b))
  d_rgb = max((x[:, :3] - y[:, :3]).abs().max().item() for x, y in zip(px_pc, px_b))
  n_rays = len(path) * H * W
  ms_pc, ms_b = 1e3 * min(t_pc), 1e3 * min(t_b)
  pools = [(pb["src_cameras"].shape[1], pb["static_src_cameras"].shape[1]) for _, pb in pooled]
  print(json.dumps({
      "what": "bullet-time sweep: %d target cameras at %dx%d, 7+3 dynamic / 15 static slots, %d samples, chunk %d, "
              "%s" % (len(path), W, H, a.samples, a.chunk, a.precision),
      "groups": [hi - lo for lo, hi in groups], "pools_dy_st": pools,
      "per_camera": {"rays_per_s": n_rays / (ms_pc / 1e3), "ms_per_sweep": ms_pc, "ms_all_reps": [1e3 * x for x in t_pc],
                     "encoder_ms": 1e3 * min(e_pc), "encoder_share": 1e3 * min(e_pc) / ms_pc},
      "batched": {"rays_per_s": n_rays / (ms_b / 1e3), "ms_per_sweep": ms_b, "ms_all_reps": [1e3 * x for x in t_b],
                  "encoder_ms": 1e3 * min(e_b), "encoder_share": 1e3 * min(e_b) / ms_b},
      "speedup": ms_pc / ms_b, "max_abs_diff_rgb_depth": d, "max_abs_diff_rgb": d_rgb,
      "pixels_bit_identical": d == 0.0,
      "timing": "wall clock of the whole sweep between device synchronisations, best of the reps; encoder passes "
                "of one sweep timed separately",
      "gpu": gpu_info(dev.index),
  }))


if __name__ == "__main__":
  main()
