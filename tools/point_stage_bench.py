"""Times the fused per-point stage (point_fused_wg_kernel: point1 -> ray-transformer attention -> point2) one
instantiation at a time, at the shapes bench.py renders: the static and the dynamic net, 8192 rays x 64 samples
(the coarse pass) and 8192 rays x 128 samples (the fine pass).

bench.py's `point1` kernel class mixes all four instantiations.  Here each runs alone through
dyn_debug_point_chain (the product kernel, no captures) on seeded pooled features G and nvalid, and its device time
is read from the library's per-launch CUDA events (dyn_profile_enable / dyn_profile_read, class point1), which
bracket the kernel only, not the hook's fp32 conversions.  Prints one JSON line per instantiation and one with the
card: ms per launch and algorithmic TFLOP/s (MACs per point from the layer widths: 147 712 for point1,
2 S 128 for the attention, 135 104 / 49 280 for the dynamic / static point2).

  python tools/point_stage_bench.py [--rays 8192] [--launches 20] [--warmup 3]
"""

import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynibar_b200 import _lib, synthetic, weights  # noqa: E402

PROF_POINT1 = 3  # bench.py: KERNEL_CLASSES.index("point1")
MAC_POINT1 = 257 * 256 + 256 * 128 + 3 * 128 * 128
MAC_POINT2 = {"dynamic": 135104, "static": 49280}


def card():
  q = "name,power.limit,clocks.sm,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = ""
  return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if out else {"name": torch.cuda.get_device_name()}


def inputs(R, S, seed, dev):
  """Seeded pooled features G [P, 272] (bf16 values, the bias columns 264, 265 = 1), nvalid [P] in {0, 1, 2, 8},
  sample points [P, 3] and ray directions [R, 3]."""
  g = torch.Generator().manual_seed(seed)
  P = R * S
  G = torch.zeros(P, 272)
  G[:, :128] = torch.randn(P, 128, generator=g) * 0.5
  G[:, 128:256] = torch.randn(P, 128, generator=g).abs() * 0.2
  G[:, 256] = torch.rand(P, generator=g) / 8
  G[:, 264:266] = 1.0
  nvalid = torch.tensor([0.0, 1.0, 2.0, 8.0])[torch.randint(0, 4, (P,), generator=g)]
  pts = torch.randn(P, 3, generator=g) * 2
  ray_dir = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
  return [t.to(torch.bfloat16).float().to(dev) if t is G else t.to(dev) for t in (G, nvalid, pts, ray_dir)]


def main():
  ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
  ap.add_argument("--rays", type=int, default=8192)
  ap.add_argument("--launches", type=int, default=20)
  ap.add_argument("--warmup", type=int, default=3)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit("point_stage_bench.py needs a GPU")
  dev = torch.device("cuda:0")
  model, _ = synthetic.make_model(64, 0, mono=True, seed=4)
  print(json.dumps({"card": card()}), flush=True)
  for kind in ("static", "dynamic"):
    net = (model.net_coarse_dy if kind == "dynamic" else model.net_coarse_st).to(dev)
    packed = weights.packed_of(net, dev)
    for S in (64, 128):
      R, P = a.rays, a.rays * S
      G, nvalid, pts, ray_dir = inputs(R, S, seed=S, dev=dev)
      out_a = torch.empty(P, 128 if kind == "static" else 4, device=dev)
      out_b = torch.empty(P, device=dev)
      pws = torch.zeros(S * 128, device=dev)

      def launch():
        _lib.check(_lib.lib.dyn_debug_point_chain(
            packed.handle, G.data_ptr(), nvalid.data_ptr(), pts.data_ptr(), ray_dir.data_ptr(), R, S,
            None, None, None, None, None, out_a.data_ptr(), out_b.data_ptr(), pws.data_ptr(), _lib.stream()))

      for _ in range(a.warmup):
        launch()
      torch.cuda.synchronize()
      _lib.lib.dyn_profile_enable(1)
      for _ in range(a.launches):
        launch()
      torch.cuda.synchronize()
      tot, n = ctypes.c_float(), ctypes.c_int()
      _lib.check(_lib.lib.dyn_profile_read(PROF_POINT1, ctypes.byref(tot), ctypes.byref(n)))
      _lib.lib.dyn_profile_enable(0)
      if n.value != a.launches:
        sys.exit("expected %d point1 launches, the profiler saw %d" % (a.launches, n.value))
      ms = tot.value / n.value
      mac = P * (MAC_POINT1 + 2 * S * 128 + MAC_POINT2[kind])
      print(json.dumps({"net": kind, "rays": R, "S": S, "keys": 128 if S == 128 else 64, "ms_per_launch": ms,
                        "tflops": 2 * mac / (ms / 1e3) / 1e12, "launches": n.value,
                        "clocks.sm_after": card().get("clocks.sm")}), flush=True)


if __name__ == "__main__":
  main()
