#!/usr/bin/env python
"""Timing of one training step of render_rays_mv's fine stage (DynibarFF) and the cost of a trainable trajectory basis.

  python tools/train_mv_bench.py [--steps 10] [--warmup 3] [--rays 1024] [--precision bf16] [--repeats 3]

Line "mv_fine_step": synthetic 512x288 scene, 7 dynamic + 11 static source views, 64 coarse + 64 fine samples, N_rand
rays.  One step = feature_net_fine forward over the 18 source images, render_rays_mv with a trainable fine stage (the
coarse stage and its encoder frozen, under no_grad), a stand-in loss (rgb + optical flows + exp_sf), backward, and
Adam over net_fine_dy / net_fine_st / motion_mlp_fine / feature_net_fine / trajectory_basis_fine.  The step time is
split with CUDA events into coarse (no grad: coarse encoder + coarse pass), fine forward (fine encoder + resampling +
fine pass + loss), backward and Adam.

Line "mono_basis_cost": the training step of bench.py's train_step line (encoder + render_rays_mono is_train=True,
1024 rays x 64 samples) with trajectory_basis frozen and with it trainable (its own Adam group at lr * 0.25, as
ibrnet/model.py:331-351), timed in alternating windows.

Prints the card's name, power limit and SM clocks of the same run, then one JSON line per measurement.
"""

import argparse
import json
import os
import subprocess
import sys

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


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


def _events(n):
  return [torch.cuda.Event(enable_timing=True) for _ in range(n)]


def mv_fine_step(dev, precision, rays, steps, warmup):
  from dynibar_b200 import feature_network, render_ray as rr, synthetic
  from dynibar_b200.projection import Projector
  N_s, N_i, V_dy, V_st = 64, 64, 7, 11
  batch, _, _, frame, t, offs = synthetic.make_scene(H=288, W=512, V_dy=V_dy, V_st=V_st, seed=3, rays=rays)
  model, args = synthetic.make_model(N_s, N_i, seed=3)
  model = synthetic.model_to(model, dev)
  model.trajectory_basis_fine = model.trajectory_basis_fine.detach().requires_grad_(True)
  torch.manual_seed(5)
  enc_c = feature_network.ResNet().to(dev).requires_grad_(False)  # feature_net: coarse stage, not trained here
  enc_f = feature_network.ResNet().to(dev).requires_grad_(True)   # feature_net_fine
  params = list(enc_f.parameters())
  for m in (model.net_fine_dy, model.net_fine_st, model.motion_mlp_fine):
    m.requires_grad_(True)
    params += list(m.parameters())
  lr = 5e-4
  opt = torch.optim.Adam([{"params": params, "lr": lr}, {"params": [model.trajectory_basis_fine], "lr": lr * 0.25}])
  b = synthetic.to_device(batch, dev)
  imgs = [b[k][0].permute(0, 3, 1, 2).contiguous() for k in ("src_rgbs", "static_src_rgbs")]
  target = torch.rand(rays, 3, device=dev)
  proj = Projector(dev)
  g = torch.Generator(device=dev).manual_seed(9)
  marks = {}
  orig_resample = rr.resample_depths

  def resample_marked(*a, **k):  # the end of the coarse pass inside render_rays_mv
    if "coarse_end" in marks:
      marks["coarse_end"].record()
    return orig_resample(*a, **k)

  def step(ev=None):
    rec = (lambda i: ev[i].record()) if ev is not None else (lambda i: None)
    if ev is not None:
      marks["coarse_end"] = ev[3]
    opt.zero_grad(set_to_none=True)
    rec(0)
    with rr.precision_scope(precision):
      with torch.no_grad():
        fc = tuple(enc_c(im)[0] for im in imgs)
      rec(1)
      ff = tuple(enc_f(im)[1] for im in imgs)
      rec(2)
      ret = rr.render_rays_mv(frame, t, offs, b, model, proj, (fc[0], None, fc[1]), (ff[0], None, ff[1]), N_s, args,
                              inv_uniform=True, N_importance=N_i, det=False, is_train=True,
                              jitter=torch.rand(rays, N_s, device=dev, generator=g),
                              u=torch.rand(rays, N_i, device=dev, generator=g))
    out = ret["outputs_fine_ref"]
    loss = ((out["rgb"] - target) ** 2).mean() + ((ret["outputs_fine_ref_dy"]["rgb"] - target) ** 2).mean()
    loss = loss + 1e-3 * out["render_flows"].abs().mean() + 1e-2 * out["exp_sf"].abs().mean()
    rec(4)
    loss.backward()
    rec(5)
    opt.step()
    rec(6)
    marks.pop("coarse_end", None)
    return loss

  rr.resample_depths = resample_marked
  try:
    for _ in range(warmup):
      step()
    torch.cuda.synchronize()
    e0, e1 = _events(2)
    e0.record()
    for _ in range(steps):
      loss = step()
    e1.record()
    torch.cuda.synchronize()
    total = e0.elapsed_time(e1) / steps
    split = dict(coarse=0.0, fine_forward=0.0, backward=0.0, adam=0.0)
    for _ in range(steps):  # a second window with phase events (their records add a little host time)
      ev = _events(7)
      step(ev)
      torch.cuda.synchronize()
      split["coarse"] += ev[0].elapsed_time(ev[1]) + ev[2].elapsed_time(ev[3])
      split["fine_forward"] += ev[1].elapsed_time(ev[2]) + ev[3].elapsed_time(ev[4])
      split["backward"] += ev[4].elapsed_time(ev[5])
      split["adam"] += ev[5].elapsed_time(ev[6])
  finally:
    rr.resample_depths = orig_resample
  return {"what": "mv_fine_step: feature_net_fine + render_rays_mv fine stage forward + backward + Adam, N_rand %d, "
                  "%d + %d samples, %d + %d views, 512x288" % (rays, N_s, N_i, V_dy, V_st),
          "precision": precision, "ms_per_step": total, "rays_per_s": rays / total * 1e3,
          "split_ms": {k: v / steps for k, v in split.items()}, "loss_last": loss.item()}


def mono_basis_cost(dev, precision, rays, steps, warmup, repeats):
  from dynibar_b200 import feature_network, render_ray as rr, synthetic
  from dynibar_b200.projection import Projector

  def setup(basis_grad):
    batch, _, _, frame, t, offs = synthetic.make_scene(H=288, W=512, V_dy=8, V_st=8, num_vv=2, seed=3, rays=rays,
                                                       anchor_offset=2)
    args = synthetic.make_args(1, 1, 0)
    model, args = synthetic.make_model(64, 0, args=args, seed=3, mono=True)
    model = synthetic.model_to(model, dev)
    params = []
    for m in (model.net_coarse_dy, model.net_coarse_st, model.motion_mlp):
      m.requires_grad_(True)
      params += list(m.parameters())
    torch.manual_seed(5)
    enc = feature_network.ResNet().to(dev).requires_grad_(True)
    groups = [{"params": params + list(enc.parameters()), "lr": 1e-4}]
    if basis_grad:
      model.trajectory_basis = model.trajectory_basis.detach().requires_grad_(True)
      groups.append({"params": [model.trajectory_basis], "lr": 1e-4 * 0.25})
    opt = torch.optim.Adam(groups)
    b = synthetic.to_device(batch, dev)
    imgs = [b[k][0].permute(0, 3, 1, 2).contiguous() for k in ("src_rgbs", "anchor_src_rgbs", "static_src_rgbs")]
    target = torch.rand(rays, 3, device=dev)
    proj = Projector(dev)

    def step():
      opt.zero_grad(set_to_none=True)
      with rr.precision_scope(precision):
        fm = tuple(enc(im)[0] for im in imgs)
        ret = rr.render_rays_mono(frame, t, offs, b, model, fm, proj, 64, args, inv_uniform=True, det=False,
                                  is_train=True, num_vv=2)
      loss = ((ret["outputs_coarse_ref"]["rgb"] - target) ** 2).mean()
      loss = loss + ((ret["outputs_coarse_anchor"]["rgb"] - target) ** 2).mean()
      loss = loss + 1e-3 * ret["outputs_coarse_ref"]["render_flows"].abs().mean()
      loss = loss + 1e-2 * ret["outputs_coarse_anchor"]["sf_seq"].abs().mean()
      loss.backward()
      opt.step()
    return step

  arms = {"basis_frozen": setup(False), "basis_trained": setup(True)}
  for fn in arms.values():
    for _ in range(warmup):
      fn()
  times = {k: [] for k in arms}
  for _ in range(repeats):
    for name, fn in arms.items():
      torch.cuda.synchronize()
      e0, e1 = _events(2)
      e0.record()
      for _ in range(steps):
        fn()
      e1.record()
      torch.cuda.synchronize()
      times[name].append(e0.elapsed_time(e1) / steps)
  return {"what": "mono_basis_cost: bench.py train_step shape (encoder + render_rays_mono is_train=True, N_rand %d, "
                  "64 samples) with trajectory_basis frozen / trained, alternating windows of %d steps" % (rays, steps),
          "precision": precision, "ms_per_step": times,
          "median_ms": {k: sorted(v)[len(v) // 2] for k, v in times.items()}}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=10)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--rays", type=int, default=1024)
  ap.add_argument("--precision", default="bf16", choices=["fp32", "bf16"])
  ap.add_argument("--repeats", type=int, default=3, help="alternating windows per arm of the mono comparison")
  a = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit("train_mv_bench: needs a CUDA device (there is no CPU timing)")
  dev = torch.device("cuda:0")
  import bench
  clocks = bench.ClockSampler(0)
  clocks.start()
  try:
    lines = [mv_fine_step(dev, a.precision, a.rays, a.steps, a.warmup),
             mono_basis_cost(dev, a.precision, a.rays, a.steps, a.warmup, a.repeats)]
  finally:
    clk = clocks.finish()
  hw = dict(card(), sm_clock_median_mhz=clk.get("sm_mhz"), throttle=clk.get("reasons"))
  print("card: %s" % json.dumps(hw))
  for line in lines:
    print(json.dumps(dict(line, card=hw)))


if __name__ == "__main__":
  main()
