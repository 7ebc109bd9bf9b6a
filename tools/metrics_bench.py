"""Times the scoring of one time step of eval_nvidia.py (11 cameras at 288 x 512 with a dynamic mask) on the GPU
against what the reference does on the host: per camera 3 SSIM + 3 PSNR, here with the float32 scipy restatement of
skimage's SSIM (tests/metrics_ref.py; scikit-image itself is not a dependency).

  python tools/metrics_bench.py [--rounds 7] [--reps 50] [--out result.json]

Three arms, each timed in alternating windows and reported as medians:
  resident  score_views on device-resident pred / gt / mask (CUDA events)
  host      score_views from host numpy arrays, as eval holds them after the device->host copy, uploads included
            (CUDA events around work that ends with the scores on the device)
  cpu       the reference's per-camera scoring on this host's CPU (wall clock), with the core count stated
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from dynibar_b200 import metrics  # noqa: E402
import metrics_ref as mr  # noqa: E402

K, H, W = 11, 288, 512


def event_ms(fn, reps):
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  start.record()
  for _ in range(reps):
    fn()
  end.record()
  end.synchronize()
  return start.elapsed_time(end) / reps


def cpu_step(pred, gt, dyn):
  """eval_nvidia.py:383-448 for every camera: valid mask, masking, 3 SSIM (the same map recomputed each time, as the
  reference's calculate_ssim does) and 3 float64 PSNR."""
  for k in range(K):
    valid = np.tile(np.float32(np.sum(pred[k], axis=-1, keepdims=True) > 1e-3), (1, 1, 3))
    g, p = gt[k] * valid, pred[k] * valid
    for m in (valid, dyn[k], 1 - dyn[k]):
      mr.calculate_ssim32(g, p, m)
      mr.calculate_psnr(g, p, m)


def card():
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except Exception as e:  # noqa: BLE001
    q = "nvidia-smi unavailable: %s" % e
  return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--rounds", type=int, default=7)
  ap.add_argument("--reps", type=int, default=50)
  ap.add_argument("--cpu-reps", type=int, default=2)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("metrics_bench: needs a CUDA device")
  dev = torch.device("cuda:0")
  pred, gt, dyn = mr.eval_case(K, H, W, seed=0)
  d_pred, d_gt, d_dyn = (torch.from_numpy(a).to(dev) for a in (pred, gt, dyn))
  resident = lambda: metrics.score_views(d_pred, d_gt, d_dyn)
  host = lambda: metrics.score_views(pred, gt, dyn)
  got = resident().cpu().numpy()
  want = np.stack([mr.eval_scores(pred[k], gt[k], dyn[k]) for k in range(K)])
  agree = float(np.abs(got - want).max())

  def cpu():
    t0 = time.perf_counter()
    for _ in range(args.cpu_reps):
      cpu_step(pred, gt, dyn)
    return (time.perf_counter() - t0) / args.cpu_reps * 1e3

  for fn in (resident, host):
    event_ms(fn, 5)
  cpu_step(pred, gt, dyn)
  ts = {"resident": [], "host": [], "cpu": []}
  for _ in range(args.rounds):
    ts["resident"].append(event_ms(resident, args.reps))
    ts["host"].append(event_ms(host, args.reps))
    ts["cpu"].append(cpu())
  # kernel time of one call (torch.profiler, a separate window after the timed ones)
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(10):
      resident()
    torch.cuda.synchronize()
  kern = {}
  for ev in prof.key_averages():
    if ev.device_type.name == "CUDA":
      kern[ev.key] = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 10 / 1e3
  med = {k: statistics.median(v) for k, v in ts.items()}
  res = {"metric": "eval_scores", "cameras": K, "size": [H, W], "rows": 3,
         "step_ms": {"gpu_resident": med["resident"], "gpu_from_host": med["host"], "cpu_float32_restatement":
                     med["cpu"], "windows": ts},
         "cpu_cores": os.cpu_count(), "input_mb": 3 * K * H * W * 3 * 4 / 1e6,
         "max_abs_err_vs_restatement": agree,
         "kernel_ms": {"total": sum(kern.values()), "by_kernel": kern}, **card()}
  line = json.dumps(res)
  print(line)
  if args.out:
    with open(args.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
