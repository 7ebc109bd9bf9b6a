#!/usr/bin/env python
"""Phase profile of the warpgroup per-view kernel (csrc/view_wg.cu) on one benchmark chunk.

  python tools/view_phases.py [--view-kernel default]

Renders one 8192-ray chunk of the bench.py scene (64 + 64 samples, 8 + 8 views, bf16) with the clock64 hook
(dyn_debug_set_view_timestamps) on, and prints for each net the phases of block 0's warpgroups, accumulated over
all iterations of the net's last launch (the second half of the fine pass), as shares of each warpgroup's
lifetime; the card's name, power limit and SM clock are read in the same run.  Needs a GPU.
"""

import argparse
import os
import sys

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

PER_NET = 616  # dyn_debug_set_view_timestamps: static net [0, 616), dynamic net [616, 1232)
SLOTS = 32
# enum Phase in csrc/view_wg.cu
PHASES = ["front end", "named-barrier waits", "weight-ring waits",
          "ray_dir_fc.0 MMA", "ray_dir_fc.0 epilogue", "ray_dir_fc.2 MMA", "ray_dir_fc.2 epilogue + feat pooling",
          "base_fc.0 MMA", "base_fc.0 epilogue", "base_fc.2 MMA", "base_fc.2 epilogue", "vis_fc.0 MMA",
          "vis_fc.0 epilogue", "vis_fc.2 MMA", "vis_fc.2 epilogue", "vis_fc2.0 MMA", "vis_fc2.0 epilogue",
          "second pooling + outputs", "front-end handoff waits"]
ITERS, LIFE = 30, 31
ROLES = ["consumer 0", "consumer 1", "front end"]


def card():
  name = torch.cuda.get_device_name(0)
  try:
    import pynvml
    pynvml.nvmlInit()
    h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
    return dict(name=name, power_limit_w=pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0,
                sm_mhz=pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM),
                sm_max_mhz=pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM))
  except Exception as e:  # NVML missing: say so instead of numbers
    return dict(name=name, nvml_error=repr(e))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--rays", type=int, default=8192, help="rays of the chunk (bench.py's chunk size)")
  a = ap.parse_args()
  assert torch.cuda.is_available(), "view_phases.py needs a GPU"
  import bench
  from dynibar_b200 import _lib, render_ray as rr, synthetic
  from dynibar_b200.projection import Projector
  w = bench.WORKLOAD
  dev = torch.device("cuda", 0)
  batch, feat_c, feat_f, frame, t, offs, model, args = bench.build_scene(a.rays)
  model = synthetic.model_to(model, dev)
  b = synthetic.to_device(batch, dev)
  fc, ff = synthetic.to_device(feat_c, dev), synthetic.to_device(feat_f, dev)
  proj = Projector(dev)
  rr.set_precision("bf16")

  def render():
    rr.new_frame()
    rr.render_rays_mv(frame, t, offs, b, model, proj, fc, ff, w["N_samples"], args, inv_uniform=True,
                      N_importance=w["N_importance"], det=True, is_train=False)

  render()  # warm-up: module load, frame packing
  buf = torch.zeros(2 * PER_NET, dtype=torch.int64, device=dev)
  _lib.lib.dyn_debug_set_view_timestamps(buf.data_ptr())
  try:
    render()
    torch.cuda.synchronize()
  finally:
    _lib.lib.dyn_debug_set_view_timestamps(None)
  c = card()
  print("card: %s" % c)
  d = buf.cpu().tolist()
  for net, base in (("static", 0), ("dynamic", PER_NET)):
    print("\n%s net (block 0; shares of each warpgroup's lifetime)" % net)
    cols = []
    for wg, role in enumerate(ROLES):
      s = d[base + SLOTS * wg: base + SLOTS * (wg + 1)]
      if s[LIFE] > 0:
        cols.append((role, s))
    print("%-40s" % "phase" + "".join("%14s" % r for r, _ in cols))
    for i, ph in enumerate(PHASES):
      if any(s[i] for _, s in cols):
        print("%-40s" % ph + "".join("%13.1f%%" % (100.0 * s[i] / s[LIFE]) for _, s in cols))
    print("%-40s" % "sum of phases" + "".join("%13.1f%%" % (100.0 * sum(s[:len(PHASES)]) / s[LIFE])
                                               for _, s in cols))
    print("%-40s" % "iterations" + "".join("%14d" % s[ITERS] for _, s in cols))
    print("%-40s" % "cycles per iteration" + "".join("%14.0f" % (s[LIFE] / max(s[ITERS], 1)) for _, s in cols))
  return 0


if __name__ == "__main__":
  sys.exit(main())
