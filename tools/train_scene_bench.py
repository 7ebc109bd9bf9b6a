#!/usr/bin/env python
"""What feeding a monocular training step costs: the reference's data loader against the device-resident scene.

  python tools/train_scene_bench.py [--steps 5] [--windows 3] [--batches 40] [--workers 16]

Writes a seeded synthetic scene (tests/mono_scene_ref.py) at 288x512 with 60 frames in a temporary directory and uses
the shipped config's view counts (configs/train_kid-running.txt: num_source_views 7, max_range 42, num_vv 3,
mask_src_view, erosion_radius 3, N_rand 3072, 64 samples).  Two feeds:

  host:   the reference's __getitem__ restated on the files (PNG / npy / npz decoding, cv2 resizes, scipy erosion) as a
          torch Dataset under a DataLoader with `workers` worker processes and pin_memory, then
          RaySamplerSingleImage(train_data, device).random_sample, as train.py:234-262 does;
  device: dynibar_b200.mono_scene.MonocularScene.sample.

Reported: the scene's load time and nbytes; per-batch time of each feed (host: the loader's next item plus
random_sample, device: sample, each up to a synchronised device); the full training step (encoder on the three stacks,
render_rays_mono is_train=True, mono_step_loss, backward, Adam; bf16) fed by each, in alternating windows of `steps`
steps; the card's name and power limit read in the same run.  Needs a GPU.
"""

import argparse
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

import mono_scene_ref as msr  # noqa: E402

N, H, W = 60, 288, 512
CFG = dict(training_height=H, num_source_views=7, max_range=42, num_vv=3, mask_src_view=True, erosion_radius=3,
           init_decay_epoch=400)


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


class HostDataset(torch.utils.data.Dataset):
  """MonocularDataset.__getitem__ on the files: every image, mask, disparity and flow read and decoded per item."""

  def __init__(self, path, cams):
    self.path, self.cams = path, cams

  def __len__(self):
    return N

  def __getitem__(self, _):
    p, c = self.path, self.cams
    rng = np.random  # the reference draws from the process's global numpy stream
    ids = msr.draw_ids(rng, N, 0, CFG, c["c2w"])
    i, a = ids["idx"], ids["anchor"]
    img = lambda j: msr.imread(os.path.join(p, "images_%dx%d" % (W, H), "%05d.png" % j))
    vv = lambda j, v: msr.imread(os.path.join(p, "source_virtual_views_%dx%d" % (W, H), "%05d" % j, "%02d.png" % v))
    dmask = lambda j: msr.imread(os.path.join(p, "dynamic_masks", "%d.png" % j))
    f32 = lambda x: x.astype(np.float32) / np.float32(255.0)
    cam = lambda c2w, K: np.concatenate(([H, W], K.flatten(), c2w.flatten())).astype(np.float32)
    src = [f32(img(j)) for j in ids["nearest"]] + [f32(vv(i, v)) for v in ids["vv"]]
    anc = [f32(img(j)) for j in ids["anchor_nearest"]] + [f32(vv(a, v)) for v in ids["anchor_vv"]]
    st = [f32(img(j)) * msr.source_mask(dmask(j), H, W) for j in ids["static"]]
    flows, masks = [], []
    for o in (1, 2, 3, -1, -2, -3):
      z = np.load(os.path.join(p, "flow_i%d" % abs(o), "%05d_%s.npz" % (i, "fwd" if o > 0 else "bwd")))
      flows.append(z["flow"])
      masks.append(np.float32(z["mask"]))
    t = torch.from_numpy
    return dict(
        id=i, anchor_id=a, num_frames=N, ref_time=float(i / float(N)), anchor_time=float(a / float(N)),
        nearest_pose_ids=t(np.array(ids["nearest"])), anchor_nearest_pose_ids=t(np.array(ids["anchor_nearest"])),
        rgb=t(f32(img(i))), disp=t(np.load(os.path.join(p, "disp", "%05d.npy" % i)) / np.float32(c["scale"])),
        motion_mask=t(msr.motion_mask(dmask(i), H, W, CFG["erosion_radius"])),
        static_mask=t(msr.static_mask(msr.imread(os.path.join(p, "static_masks", "%d.png" % i)), H, W)),
        flows=t(np.stack(flows)), masks=t(np.stack(masks)), camera=t(cam(c["c2w"][i], c["K"][i])),
        anchor_camera=t(cam(c["c2w"][a], c["K"][a])), rgb_path=c["rgb_files"][i], src_rgbs=t(np.stack(src)),
        src_cameras=t(np.stack([cam(c["c2w"][j], c["K"][j]) for j in ids["nearest"]] +
                               [cam(c["vv_c2w"][i, v], c["K"][i]) for v in ids["vv"]])),
        static_src_rgbs=t(np.stack(st)), static_src_cameras=t(np.stack([cam(c["c2w"][j], c["K"][j])
                                                                         for j in ids["static"]])),
        anchor_src_rgbs=t(np.stack(anc)),
        anchor_src_cameras=t(np.stack([cam(c["c2w"][j], c["K"][j]) for j in ids["anchor_nearest"]] +
                                      [cam(c["vv_c2w"][a, v], c["K"][i]) for v in ids["anchor_vv"]])),
        depth_range=t(c["depth_range"]))


def _next(it, loader):
  try:
    return next(it[0])
  except StopIteration:
    it[0] = iter(loader)
    return next(it[0])


def _stats(v):
  s = sorted(v)
  return {"windows_ms": [round(x, 3) for x in v], "median_ms": round(s[len(s) // 2], 3),
          "spread_ms": round(s[-1] - s[0], 3)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=5)
  ap.add_argument("--windows", type=int, default=3)
  ap.add_argument("--batches", type=int, default=40)
  ap.add_argument("--workers", type=int, default=16)
  ap.add_argument("--rays", type=int, default=3072, help="N_rand of the batches")
  ap.add_argument("--step-rays", type=int, default=1024,
                  help="rays of the timed training steps (3072 rays x 64 samples with 14 static views does not fit "
                       "the training path's saved activations in 80 GB)")
  a = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit("train_scene_bench: needs a CUDA device")
  from dynibar_b200 import criterion as cr, feature_network, mono_scene, render_ray as rr, sample_ray, synthetic
  from dynibar_b200.projection import Projector
  dev = torch.device("cuda:0")
  args_s = SimpleNamespace(**CFG)
  with tempfile.TemporaryDirectory() as tmp:
    path = msr.write_scene(os.path.join(tmp, "scene", "dense"), msr.synthetic_scene(3, N, H, W, levels=256))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    scene = mono_scene.MonocularScene(path, args_s, dev)
    torch.cuda.synchronize()
    load_s = time.perf_counter() - t0
    loader = torch.utils.data.DataLoader(HostDataset(path, scene.cams), batch_size=1, shuffle=True,
                                         num_workers=a.workers, pin_memory=True, persistent_workers=True,
                                         prefetch_factor=2)
    it = [iter(loader)]

    def host_batch_rays():
      td = _next(it, loader)
      return td, sample_ray.RaySamplerSingleImage(td, dev).random_sample(a.rays, "center")

    rng = np.random.RandomState(0)

    def dev_batch():
      return scene.sample(rng, a.rays, "center")

    # per-batch time, each up to a synchronised device
    per_batch = {}
    for name, fn in (("host", host_batch_rays), ("device", dev_batch)):
      for _ in range(3):
        fn()
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      for _ in range(a.batches):
        fn()
      torch.cuda.synchronize()
      per_batch[name] = (time.perf_counter() - t0) * 1e3 / a.batches

    print("scene load %.2f s, %.1f MB; batch ms %s" % (load_s, scene.nbytes / 1e6, per_batch), flush=True)

    # full training steps fed by each
    host_step = lambda: (lambda td: (td, sample_ray.RaySamplerSingleImage(td, dev).random_sample(a.step_rays,
                                                                                                "center")))(
        _next(it, loader))
    dev_step = lambda: scene.sample(rng, a.step_rays, "center")
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

    def step(feed):
      td, b = feed()
      i, an = int(td["id"]), int(td["anchor_id"])  # train.py:239-240 reads the ids on the host
      offs = ([int(j) - i for j in td["nearest_pose_ids"][0]], [int(j) - an for j in td["anchor_nearest_pose_ids"][0]])
      with rr.precision_scope("bf16"):
        fm = tuple(enc(b[k][0].permute(0, 3, 1, 2).contiguous())[0]
                   for k in ("src_rgbs", "anchor_src_rgbs", "static_src_rgbs"))
        ret = rr.render_rays_mono((i, an), (td["ref_time"].to(dev), td["anchor_time"].to(dev)), offs, b, model, fm,
                                  proj, 64, args, inv_uniform=True, det=False, is_train=True, num_vv=3)
        loss, _ = cr.mono_step_loss(ret, b, args, 0)
      opt.zero_grad(set_to_none=True)
      loss.backward()
      opt.step()

    feeds = {"host": host_step, "device": dev_step}
    for f in feeds.values():
      for _ in range(2):
        step(f)
    times = {k: [] for k in feeds}
    for _ in range(a.windows):
      for k, f in feeds.items():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.steps):
          step(f)
        torch.cuda.synchronize()
        times[k].append((time.perf_counter() - t0) * 1e3 / a.steps)
    hw = card()
    print("card: %s" % json.dumps(hw))
    print(json.dumps({
        "what": "monocular training feed, 288x512, %d frames, N_rand %d (training steps: %d rays), 7 source views, "
                "num_vv 3, mask_src_view, erosion_radius 3; host = DataLoader(%d workers, pin_memory) + random_sample"
                % (N, a.rays, a.step_rays, a.workers),
        "scene_load_s": round(load_s, 3), "scene_nbytes": int(scene.nbytes),
        "batch_ms": {k: round(v, 3) for k, v in per_batch.items()},
        "step": {k: _stats(v) for k, v in times.items()}, "card": hw}))
    del loader, it


if __name__ == "__main__":
  main()
