#!/usr/bin/env python
"""What a monocular training step costs whole and in ray slices (dynibar_b200.train_step.mono_step_backward).

  python tools/train_step_bench.py [--steps 5] [--windows 3]

The seeded synthetic scene of tools/train_scene_bench.py (288x512, 60 frames, the shipped config's view counts: 7
source + 3 virtual dynamic views, 14 static views, 64 samples), fed by the device-resident scene; bf16, the full
criterion at epoch 0, the encoder forward and backward on the three stacks, Adam.  Arms, timed in alternating windows
of `steps` steps (each up to a synchronised device):
  a  1024 rays: render_rays_mono(is_train=True), mono_step_loss, backward (train.py's sequence)
  b  1024 rays: mono_step_backward(slice_rays=1024) -- one slice, the same sequence
  c  1024 rays: mono_step_backward(slice_rays=512)
  d  3072 rays: mono_step_backward(slice_rays=1024) -- the shipped N_rand
Reported per arm: ms per step (median and spread of the windows), peak torch.cuda.max_memory_allocated (reset before
the arm's first window), and for the sliced arms pass 1's share of the step (pass 1 timed alone on the same batches,
train_step.batch_table over the step's slices); the card's name, power limit and SM clock read in the same run.
Needs a GPU.
"""

import json
import os
import subprocess
import sys
import tempfile
import time
from types import SimpleNamespace

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
  if p not in sys.path:
    sys.path.insert(0, p)

import argparse  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

import mono_scene_ref as msr  # noqa: E402

N, H, W = 60, 288, 512
CFG = dict(training_height=H, num_source_views=7, max_range=42, num_vv=3, mask_src_view=True, erosion_radius=3,
           init_decay_epoch=400)
ARMS = {"a_1024_today": (1024, None), "b_1024_one_slice": (1024, 1024), "c_1024_slices_512": (1024, 512),
        "d_3072_slices_1024": (3072, 1024)}


def card():
  info = {"name": torch.cuda.get_device_name(0)}
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                          "--id=%d" % torch.cuda.current_device()], capture_output=True, text=True, timeout=30)
    power, sm, sm_max = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
    info.update(power_limit=power, sm_clock=sm, sm_max_clock=sm_max)
  except Exception as e:  # nvidia-smi missing: say so instead of guessing
    info.update(power_limit=None, sm_clock=None, sm_max_clock=None, query_error=repr(e))
  return info


def _stats(v):
  s = sorted(v)
  return {"windows_ms": [round(x, 2) for x in v], "median_ms": round(s[len(s) // 2], 2),
          "spread_ms": round(s[-1] - s[0], 2)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=5)
  ap.add_argument("--windows", type=int, default=3)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit("train_step_bench: needs a CUDA device")
  from dynibar_b200 import criterion as cr, feature_network, mono_scene, render_ray as rr, synthetic, train_step as ts
  from dynibar_b200.projection import Projector
  dev = torch.device("cuda:0")
  with tempfile.TemporaryDirectory() as tmp:
    path = msr.write_scene(os.path.join(tmp, "scene", "dense"), msr.synthetic_scene(3, N, H, W, levels=256))
    scene = mono_scene.MonocularScene(path, SimpleNamespace(**CFG), dev)
  args = synthetic.make_args(0, 1, 0)
  args = SimpleNamespace(**dict(vars(args), w_disp=1e-1, w_flow=1e-2, w_cycle=0.1, cycle_factor=0.1,
                                anneal_cycle=True, w_reg=0.05, w_skew_entropy=5e-4, w_distortion=1e-3,
                                decay_rate=10.0, init_decay_epoch=400))
  model, args = synthetic.make_model(64, 0, num_frames=N, args=args, seed=3, mono=True)
  model = synthetic.model_to(model, dev)
  params = []
  for m in (model.net_coarse_dy, model.net_coarse_st, model.motion_mlp):
    m.requires_grad_(True)
    params += list(m.parameters())
  torch.manual_seed(5)
  enc = feature_network.ResNet().to(dev).requires_grad_(True)
  opt = torch.optim.Adam(params + list(enc.parameters()), lr=1e-4)
  proj = Projector(dev)
  rng = np.random.RandomState(0)

  def inputs(rays):
    td, b = scene.sample(rng, rays, "center")
    i, an = int(td["id"]), int(td["anchor_id"])  # train.py:239-240 reads the ids on the host
    offs = ([int(j) - i for j in td["nearest_pose_ids"][0]], [int(j) - an for j in td["anchor_nearest_pose_ids"][0]])
    return (i, an), (td["ref_time"].to(dev), td["anchor_time"].to(dev)), offs, b

  def featmaps(b):
    return tuple(enc(b[k][0].permute(0, 3, 1, 2).contiguous())[0]
                 for k in ("src_rgbs", "anchor_src_rgbs", "static_src_rgbs"))

  def step(arm):
    rays, slice_rays = ARMS[arm]
    frame, t, offs, b = inputs(rays)
    opt.zero_grad(set_to_none=True)
    with rr.precision_scope("bf16"):
      fm = featmaps(b)
      if slice_rays is None:
        ret = rr.render_rays_mono(frame, t, offs, b, model, fm, proj, 64, args, inv_uniform=True, det=False,
                                  is_train=True, num_vv=3)
        loss, _ = cr.mono_step_loss(ret, b, args, 0)
        del ret
        loss.backward()
      else:
        ts.mono_step_backward(frame, t, offs, b, model, fm, proj, 64, args, 0, slice_rays=slice_rays, num_vv=3,
                              precision="bf16")
    opt.step()

  def pass1(arm):
    rays, slice_rays = ARMS[arm]
    frame, t, offs, b = inputs(rays)
    jitter = torch.rand(rays, 64, device=dev)
    with torch.no_grad(), rr.precision_scope("bf16"):
      fm = featmaps(b)
    spans = ts.slice_plan(rays, slice_rays, 64)
    render = lambda lo, hi: rr._render_mono_train(frame, t, offs, ts._slice_batch(b, lo, hi), model, fm, 64, args,
                                                  True, False, True, 3, jitter[lo:hi])
    with rr.precision_scope("bf16"):
      ts.batch_table(render, b, spans, args, 0, False)

  def timed(fn, arm):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.steps):
      fn(arm)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / a.steps

  for arm in ARMS:  # warm-up
    for _ in range(2):
      step(arm)
  times, peaks, p1 = {k: [] for k in ARMS}, {}, {k: [] for k in ARMS if ARMS[k][1] not in (None, ARMS[k][0])}
  for w in range(a.windows):
    for arm in ARMS:
      if w == 0:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
      times[arm].append(timed(step, arm))
      if w == 0:
        peaks[arm] = torch.cuda.max_memory_allocated() / 2 ** 30
      if arm in p1:
        p1[arm].append(timed(pass1, arm))
  hw = card()
  res = {}
  for arm in ARMS:
    res[arm] = dict(_stats(times[arm]), peak_GB=round(peaks[arm], 2))
    if arm in p1:
      med = sorted(p1[arm])[len(p1[arm]) // 2]
      res[arm].update(pass1_median_ms=round(med, 2), pass1_share=round(med / res[arm]["median_ms"], 3))
  print(json.dumps({"what": "monocular training step, 288x512, %d frames, 7 + 3 dynamic and 14 static views, 64 "
                            "samples, bf16, full criterion at epoch 0, encoder included, Adam; %d steps per window"
                            % (N, a.steps), "arms": res, "card": hw}))


if __name__ == "__main__":
  main()
