"""Times the virtual-source-view product on the GPU against a torch-on-GPU restatement that splats with index_add_
(float atomics; the external `splatting` extension cannot be built here, so it is not the baseline).

  python tools/virtual_views_bench.py [--frames 100] [--rounds 5] [--out result.json]

Two workloads, each timed in alternating windows (ours, torch, ours, ...) and reported as medians:
  frame  one frame's 8 views at 288 x 512 from device-resident inputs (one render_virtual_views call)
  scene  --frames frames through what tools/make_virtual_views.py does per frame, minus file I/O: cv2 resizing of a
         576 x 1024 frame on the host, upload, the 8 views, download of the uint8 views.
Prints one JSON line with the card's name and power limit beside the numbers.
"""

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynibar_b200 import virtual_views as vv  # noqa: E402

H, W = 288, 512


def torch_views(img, disp, K, ref2w, tgt_c2w):
  """The same product in torch ops on the GPU; render_forward_splat's splat by index_add_."""
  dev = img.device
  V = len(tgt_c2w)
  depth10 = (1.0 / disp) / 10.0
  p = F.pad(depth10[None, None], (1, 1, 1, 1), mode="replicate")
  kx = torch.tensor([[-1.0, 0.0, 1.0], [-2.0, 0.0, 2.0], [-1.0, 0.0, 1.0]], device=dev)
  g = F.conv2d(p, torch.stack([kx, kx.t()])[:, None])
  alpha = torch.exp(-0.5 * torch.sqrt(g[0, 0] ** 2 + g[0, 1] ** 2))
  rgba = torch.cat([img * 255.0, alpha[..., None]], -1).reshape(-1, 4)
  R, t = [], []
  for c in tgt_c2w:
    tgt2w = np.eye(4)
    tgt2w[:3, :4] = c
    T = np.dot(np.linalg.inv(tgt2w), ref2w)
    R.append(T[:3, :3])
    t.append(T[:3, 3])
  R = torch.from_numpy(np.stack(R)).float().to(dev)
  t = torch.from_numpy(np.stack(t)).float().to(dev)
  k = torch.from_numpy(np.array(K)).float()
  ki, k = k.inverse().to(dev), k.to(dev)
  ys, xs = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32),
                          torch.arange(W, device=dev, dtype=torch.float32), indexing="ij")
  coord = torch.stack([xs, ys, torch.ones_like(xs)], -1).reshape(-1, 3)
  pts = (1.0 / disp).reshape(-1, 1) * (coord @ ki.t())
  pts = torch.einsum("vij,nj->vni", R, pts) + t[:, None]
  pts = pts @ k.t()
  z = pts[..., 2]
  ox = pts[..., 0] / z.clamp(min=1e-8)
  oy = pts[..., 1] / z.clamp(min=1e-8)
  imp = 1.0 / z
  lo, hi = imp.amin(1, keepdim=True), imp.amax(1, keepdim=True)
  e = torch.exp((imp - lo) / (hi - lo + 1e-6) * 20 - 10)
  vals = torch.cat([rgba[None] * e[..., None], e[..., None]], -1).reshape(-1, 5)
  nx, ny = torch.floor(ox), torch.floor(oy)
  acc = torch.zeros(V * H * W, 5, device=dev)
  base = (torch.arange(V, device=dev) * (H * W))[:, None]
  for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
    cx, cy = nx + dx, ny + dy
    w = (1 - (ox - cx).abs()) * (1 - (oy - cy).abs())
    ok = ((cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)).reshape(-1)
    idx = (base + cy * W + cx).long().reshape(-1)
    acc.index_add_(0, idx[ok], (vals * w.reshape(-1, 1))[ok])
  Fr = (acc[:, :4] / (acc[:, 4:] + 1e-7)).reshape(V, H, W, 4)
  m = (Fr[..., 3] > 0.5).float()[:, None]
  mp = F.pad(m, (1, 1, 1, 1), mode="replicate")
  m = torch.minimum(torch.minimum(mp[..., 1:-1, 1:-1], mp[..., :-2, 1:-1]), mp[..., 2:, 1:-1])
  m = torch.minimum(torch.minimum(m, mp[..., 1:-1, :-2]), mp[..., 1:-1, 2:])[:, 0, ..., None]
  return ((255.0 * (Fr[..., :3] / 255.0).clamp(0, 1)) * m).to(torch.uint8)


def timed(fn, reps):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(reps):
    fn()
  torch.cuda.synchronize()
  return (time.perf_counter() - t0) / reps * 1e3


def card():
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except Exception as e:  # noqa: BLE001
    q = "nvidia-smi unavailable: %s" % e
  return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--frames", type=int, default=100)
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--reps", type=int, default=50)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("virtual_views_bench: needs a CUDA device")
  import cv2
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
  import virtual_views_ref as vr
  dev = torch.device("cuda:0")
  img, disp, K, ref2w, tgt = vr.frame_case()
  d_img, d_disp = torch.from_numpy(img).to(dev), torch.from_numpy(disp).to(dev)
  ours = lambda: vv.render_virtual_views(d_img, d_disp, K, ref2w, tgt)
  base = lambda: torch_views(d_img, d_disp, K, ref2w, tgt)
  agree = vr.png_mismatch(ours().cpu().numpy(), base().cpu().numpy())
  from dynibar_b200 import _lib
  _lib.lib.dyn_launch_count(1)
  ours()
  launches = _lib.lib.dyn_launch_count(0)
  ts = {"ours": [], "torch": []}
  for fn in (ours, base):
    timed(fn, 5)
  for _ in range(args.rounds):
    ts["ours"].append(timed(ours, args.reps))
    ts["torch"].append(timed(base, args.reps))

  # scene: per frame cv2 resize of a 2x frame on the host, upload, views, download
  big_img = cv2.resize(img, (2 * W, 2 * H), interpolation=cv2.INTER_LINEAR)
  big_depth = cv2.resize(1.0 / disp, (2 * W, 2 * H), interpolation=cv2.INTER_NEAREST)

  def scene(fn):
    def run():
      for _ in range(args.frames):
        i = cv2.resize(big_img, (W, H), interpolation=cv2.INTER_AREA)
        d = cv2.resize((1.0 / big_depth).astype(np.float32), (W, H), interpolation=cv2.INTER_LINEAR)
        out = fn(torch.from_numpy(i).to(dev), torch.from_numpy(d).to(dev), K, ref2w, tgt)
        out.cpu()
    return run
  s_ours, s_base = scene(vv.render_virtual_views), scene(torch_views)
  timed(s_ours, 1)
  timed(s_base, 1)
  ss = {"ours": [], "torch": []}
  for _ in range(max(3, args.rounds // 2)):
    ss["ours"].append(timed(s_ours, 1))
    ss["torch"].append(timed(s_base, 1))
  # device time of one frame's kernels (torch.profiler, a separate window after the timed ones): how much of the
  # frame time is kernel time rather than launch gaps and host work
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(10):
      ours()
    torch.cuda.synchronize()
  kern = {}
  for ev in prof.key_averages():
    if ev.device_type.name == "CUDA":
      kern[ev.key] = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 10 / 1e3
  med = {k: statistics.median(v) for k, v in ts.items()}
  smed = {k: statistics.median(v) for k, v in ss.items()}
  res = {"metric": "virtual_views", "views": len(tgt), "size": [H, W], "launches_per_frame": launches,
         "frame_ms": {"ours": med["ours"], "torch_index_add": med["torch"], "windows": ts},
         "scene_s": {"frames": args.frames, "ours": smed["ours"] / 1e3, "torch_index_add": smed["torch"] / 1e3,
                     "windows_ms": ss},
         "bytes_over_1lsb_vs_torch": agree,
         "frame_kernel_ms": {"total": sum(kern.values()), "by_kernel": kern}, **card()}
  line = json.dumps(res)
  print(line)
  if args.out:
    with open(args.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
