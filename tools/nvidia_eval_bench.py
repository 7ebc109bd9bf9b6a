#!/usr/bin/env python
"""What feeding one Nvidia-benchmark time step costs: the reference's front end against the device-resident scene.

  python tools/nvidia_eval_bench.py [--reps 5] [--eval-reps 2] [--workers 12] [--samples 16] [--out FILE]

Writes a seeded synthetic Nvidia scene (tests/nvi_scene_ref.py) at 288x512 with 24 frames, ground truth JPEGs at
1080x1920 and grey masks in a temporary directory.  Two arms, alternated:

  host:   eval_nvidia.py's front end restated: a Dataset whose items read the 18 source frames (PIL, as imageio) and the
          coarse masks under a DataLoader with `workers` worker processes, RaySamplerSingleImage(item).get_all() per
          camera, stack_ray_batches, and cv2 ground truth (INTER_AREA) and masks (INTER_NEAREST) on the host, uploaded;
  device: dynibar_b200.nvidia_scene.NvidiaScene.time_step.

Reported: the scene's load time and nbytes; one time step's inputs by each arm (up to a synchronised device); a whole
time step's evaluation (encoders, render_multi_image_nvi over the 11 cameras, score_views, read-back) fed by each arm,
with the synthetic model at `samples` + `samples` samples; the card's name and power limit read in the same run.
Needs a GPU.
"""

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
  if p not in sys.path:
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nvi_scene_ref as nsr  # noqa: E402

N, H, W = 24, 288, 512


def card():
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                        "--id=%d" % torch.cuda.current_device()], capture_output=True, text=True, timeout=30)
    return q.stdout.strip()
  except Exception as e:  # nvidia-smi missing: say so instead of guessing
    return "nvidia-smi unavailable: %r" % (e,)


class HostItems(torch.utils.data.Dataset):
  """DynamicVideoDataset(img_i): item i is camera i's, every source frame and coarse mask read again per item."""

  def __init__(self, root, img_i, cams):
    self.root, self.img_i, self.cams = root, img_i, cams

  def __len__(self):
    return nsr.CYCLE

  def __getitem__(self, i):
    c = self.cams
    return nsr.item(self.root, self.img_i, i, N, c["K"], c["c2w"], c["depth_range"], True)


def host_step(root, img_i, cams, workers, dev):
  from dynibar_b200 import sample_ray as sr
  # the items are collated already (batch dimension 1), as the reference's batch_size=1 loader yields them
  loader = torch.utils.data.DataLoader(HostItems(root, img_i, cams), batch_size=None, num_workers=workers,
                                       shuffle=False)
  items = [d for i, d in enumerate(loader) if i != img_i % nsr.CYCLE]
  samplers = [sr.RaySamplerSingleImage(d, device=dev) for d in items]
  rb, _, _ = sr.stack_ray_batches([s.get_all() for s in samplers])
  gt, dm = nsr.ground_truth(root, img_i, nsr.target_cameras(img_i), H, W)
  return rb, samplers, torch.from_numpy(gt).to(dev), torch.from_numpy(dm).to(dev), items[0]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=5)
  ap.add_argument("--eval-reps", type=int, default=2)
  ap.add_argument("--workers", type=int, default=12)
  ap.add_argument("--samples", type=int, default=16)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  assert torch.cuda.is_available(), "nvidia_eval_bench needs a GPU"
  from dynibar_b200 import metrics, nvidia_scene as ns, synthetic
  from dynibar_b200.feature_network import ResNet
  from dynibar_b200.projection import Projector
  from dynibar_b200.render_image import render_multi_image_nvi
  dev = torch.device("cuda:0")
  res = dict(card=card(), shape="%d frames of %dx%d, ground truth 1080x1920" % (N, H, W), workers=a.workers)
  with tempfile.TemporaryDirectory() as tmp:
    s = nsr.synthetic_scene(5, N, H, W, [(1080, 1920)], (540, 960), (H, W), False, levels=16)
    root = nsr.write_scene(os.path.join(tmp, "scene", "dense"), s)
    args = types.SimpleNamespace(mask_static=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    scene = ns.NvidiaScene(root, args, dev)
    torch.cuda.synchronize()
    res["load_s"], res["scene_MB"] = time.perf_counter() - t0, scene.nbytes / 1e6
    cams = ns.load_cameras(root)
    steps = scene.steps
    times = dict(host=[], device=[])
    host_step(root, steps[0], cams, a.workers, dev)  # warm up both arms
    scene.time_step(steps[0])
    for r in range(a.reps):
      img_i = steps[r % len(steps)]
      for arm in (("host", "device") if r % 2 == 0 else ("device", "host")):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if arm == "host":
          host_step(root, img_i, cams, a.workers, dev)
        else:
          scene.time_step(img_i)
        torch.cuda.synchronize()
        times[arm].append(time.perf_counter() - t0)
    res["inputs_ms"] = {k: [round(1e3 * x, 2) for x in v] for k, v in times.items()}

    model, margs = synthetic.make_model(N_samples=a.samples, N_importance=a.samples, num_frames=N, seed=0)
    model = synthetic.model_to(model, dev)
    model.feature_net = ResNet().to(dev).requires_grad_(False)
    model.feature_net_fine = ResNet().to(dev).requires_grad_(False)
    margs.chunk_size, margs.N_samples, margs.N_importance, margs.inv_uniform, margs.white_bkgd = \
        8192, a.samples, a.samples, True, False
    margs.mask_static = True
    P = Projector(dev)

    def eval_host(img_i):
      rb, samplers, gt, dm, d0 = host_step(root, img_i, cams, a.workers, dev)
      src = rb["src_rgbs"].squeeze(0).permute(0, 3, 1, 2)
      st = rb["static_src_rgbs"].squeeze(0).permute(0, 3, 1, 2)
      fc, _ = model.feature_net(src)
      _, sc = model.feature_net(st)
      ff, _ = model.feature_net_fine(src)
      _, sf = model.feature_net_fine(st * rb["static_src_masks"].squeeze(0)[:, None, ...])
      offs = [int(j - img_i) for j in d0["nearest_pose_ids"].squeeze().tolist()]
      rets = render_multi_image_nvi((img_i, None), (d0["ref_time"].to(dev), None), (offs, None), samplers, rb, model,
                                    P, margs.chunk_size, margs.N_samples, margs, inv_uniform=True,
                                    N_importance=margs.N_importance, det=True, coarse_featmaps=(fc, None, sc),
                                    fine_featmaps=(ff, None, sf), is_train=False)
      pred = torch.stack([r["outputs_fine_ref"]["rgb"] for r in rets]).to(dev)
      return metrics.score_views(pred, gt, dm).cpu().numpy()

    def eval_device(img_i):
      step = scene.time_step(img_i)
      pred = scene.render(step, model, P, margs)
      return metrics.score_views(pred, step["gt_rgb"], step["dynamic_mask"]).cpu().numpy()

    etimes, diffs = dict(host=[], device=[]), []
    with torch.no_grad():
      eval_host(steps[0]), eval_device(steps[0])
      for r in range(a.eval_reps):
        img_i = steps[(r + 1) % len(steps)]
        out = {}
        for arm in (("host", "device") if r % 2 == 0 else ("device", "host")):
          torch.cuda.synchronize()
          t0 = time.perf_counter()
          out[arm] = (eval_host if arm == "host" else eval_device)(img_i)
          torch.cuda.synchronize()
          etimes[arm].append(time.perf_counter() - t0)
        diffs.append(float(np.abs(out["host"] - out["device"]).max()))
    res["eval_step_s"] = {k: [round(x, 3) for x in v] for k, v in etimes.items()}
    res["eval_samples"] = "%d + %d" % (a.samples, a.samples)
    res["scores_max_abs_diff"] = max(diffs) if diffs else None
  line = json.dumps(res)
  print(line)
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
