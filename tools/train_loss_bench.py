#!/usr/bin/env python
"""What the training criterion costs in a step, and what the CUDA criterion changes.

  python tools/train_loss_bench.py [--steps 10] [--warmup 3] [--windows 3] [--rays 1024] [--precision bf16]

The step is bench.py's train_step (BASELINE configs[2]: 2-D encoder + render_rays_mono is_train=True, 1024 rays x 64
samples, 512x288, Adam) with the real criterion of train.py:300-456 instead of bench.py's four-term stand-in;
supervision (rgb, disp, masks, flows) comes from a seeded generator.  Two arms share the model, the optimizer state
and the batch, and are timed in alternating windows of `steps` steps within this process:

  torch: the torch restatement of the criterion (tests/loss_ref.py) applied to the library's device outputs
  cuda:  dynibar_b200.criterion.mono_step_loss

Reported: ms per step of each arm per window (CUDA events) with median and spread; the criterion's own forward +
backward time on a detached copy of one step's outputs; its kernel launches (torch.profiler, a separate pass); the
loss components of both arms on the same outputs; the card's name and power limit read in the same run.  Needs a GPU.
"""

import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
  if p not in sys.path:
    sys.path.insert(0, p)

import torch  # noqa: E402

EPOCH = 0  # every rgb term present (epoch < init_decay_epoch)
GRAD_KEYS = {"outputs_coarse_ref": ("rgb", "rgb_dy", "rgb_static", "depth", "render_flows", "weights", "weights_dy",
                                    "weights_st"),
             "outputs_coarse_ref_dy": ("rgb",), "outputs_coarse_anchor": ("rgb", "pts_traj_ref", "pts_traj_anchor",
                                                                          "sf_seq"),
             "outputs_coarse_anchor_dy": ("rgb",)}


def card():
  info = {"name": torch.cuda.get_device_name(0)}
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                          "--id=%d" % torch.cuda.current_device()], capture_output=True, text=True, timeout=30)
    power, sm_max = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
    info.update(power_limit=power, sm_max_clock=sm_max)
  except Exception as e:  # nvidia-smi missing: say so instead of guessing
    info.update(power_limit=None, sm_max_clock=None, query_error=repr(e))
  return info


def _timed(fn, n):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  e0.record()
  for _ in range(n):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / n


def _stats(v):
  s = sorted(v)
  return {"windows_ms": v, "median_ms": s[len(s) // 2], "spread_ms": s[-1] - s[0]}


def _leaves(ret):
  return {o: {k: (v.detach().clone().requires_grad_(True) if k in GRAD_KEYS.get(o, ()) else
                  (v.detach() if torch.is_tensor(v) else v)) for k, v in d.items()}
          for o, d in ret.items() if isinstance(d, dict)}


def _kernel_launches(fn):
  from torch.profiler import ProfilerActivity, profile
  fn()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  dev = getattr(torch.autograd.DeviceType, "CUDA")
  return int(sum(e.count for e in prof.key_averages() if e.device_type == dev))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=10)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--windows", type=int, default=3, help="alternating windows per arm (>= 3)")
  ap.add_argument("--rays", type=int, default=1024)
  ap.add_argument("--precision", default="bf16", choices=["fp32", "bf16"])
  a = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit("train_loss_bench: needs a CUDA device (there is no CPU timing)")
  if a.windows < 3:
    sys.exit("train_loss_bench: at least three windows per arm")
  import loss_ref
  from dynibar_b200 import criterion as cr, feature_network, render_ray as rr, synthetic
  from dynibar_b200.projection import Projector
  dev = torch.device("cuda:0")
  R, H, W = a.rays, 288, 512
  batch, _, _, frame, t, offs = synthetic.make_scene(H=H, W=W, V_dy=8, V_st=8, num_vv=2, seed=3, rays=R,
                                                     anchor_offset=2)
  args = synthetic.make_args(1, 1, 0)
  model, args = synthetic.make_model(64, 0, args=args, seed=3, mono=True)
  args = SimpleNamespace(**dict(vars(args), w_disp=5e-2, w_flow=5e-3, w_cycle=0.1, cycle_factor=0.1, anneal_cycle=False,
                                w_reg=0.05, w_skew_entropy=1e-3, w_distortion=1e-3, decay_rate=10.0,
                                init_decay_epoch=150))  # the reference's defaults (config.py)
  model = synthetic.model_to(model, dev)
  params = []
  for m in (model.net_coarse_dy, model.net_coarse_st, model.motion_mlp):
    m.requires_grad_(True)
    params += list(m.parameters())
  model.trajectory_basis = model.trajectory_basis.detach().requires_grad_(True)
  torch.manual_seed(5)
  enc = feature_network.ResNet().to(dev).requires_grad_(True)
  opt = torch.optim.Adam([{"params": params + list(enc.parameters()), "lr": 1e-4},
                          {"params": [model.trajectory_basis], "lr": 1e-4 * 0.25}])
  b = synthetic.to_device(batch, dev)
  g = torch.Generator().manual_seed(17)
  b.update({k: v.to(dev) for k, v in dict(
      rgb=torch.rand(R, 3, generator=g), disp=torch.rand(R, generator=g),
      motion_mask=(torch.rand(R, generator=g) > 0.5).float(), flows=torch.randn(6, R, 2, generator=g),
      masks=(torch.rand(6, R, 1, generator=g) > 0.3).float()).items()})
  b["static_mask"] = 1.0 - b["motion_mask"]
  imgs = [b[k][0].permute(0, 3, 1, 2).contiguous() for k in ("src_rgbs", "anchor_src_rgbs", "static_src_rgbs")]
  proj = Projector(dev)
  losses = {"torch": loss_ref.mono_step_loss, "cuda": cr.mono_step_loss}

  def forward():
    with rr.precision_scope(a.precision):
      fm = tuple(enc(im)[0] for im in imgs)
      return rr.render_rays_mono(frame, t, offs, b, model, fm, proj, 64, args, inv_uniform=True, det=False,
                                 is_train=True, num_vv=2)

  def step(arm):
    opt.zero_grad(set_to_none=True)
    loss, _ = losses[arm](forward(), b, args, EPOCH)
    loss.backward()
    opt.step()

  for arm in losses:
    for _ in range(a.warmup):
      step(arm)
  times = {arm: [] for arm in losses}
  for _ in range(a.windows):
    for arm in losses:
      times[arm].append(_timed(lambda: step(arm), a.steps))

  # ---- the criterion alone, on a detached copy of one step's outputs
  opt.zero_grad(set_to_none=True)
  ret = forward()
  alone, launches, comps = {}, {}, {}

  def loss_only(arm):
    x = _leaves(ret)

    def run():
      loss, terms = losses[arm](x, b, args, EPOCH)
      loss.backward()
      return terms
    return run

  for arm in losses:
    run = loss_only(arm)
    for _ in range(a.warmup):
      run()
    reps = [_timed(run, 20) for _ in range(a.windows)]
    alone[arm] = _stats(reps)
    comps[arm] = {k: float(v) for k, v in run().items()}
    launches[arm] = _kernel_launches(run)
  hw = card()
  print("card: %s" % json.dumps(hw))
  print(json.dumps({
      "what": "mono training step with the full criterion (encoder + render_rays_mono is_train=True + loss + backward "
              "+ Adam), N_rand %d, 64 samples, 512x288, epoch %d; arms alternate in windows of %d steps" %
              (R, EPOCH, a.steps),
      "precision": a.precision, "step": {arm: _stats(v) for arm, v in times.items()},
      "loss_forward_backward": alone, "loss_kernel_launches": launches, "components": comps, "card": hw}))


if __name__ == "__main__":
  main()
