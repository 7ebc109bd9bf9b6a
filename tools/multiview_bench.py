"""One time step of the Nvidia evaluation, rendered two ways, on the GPU.

  python tools/multiview_bench.py [--cameras 11] [--reps 2]              # 1 GPU
  torchrun --nproc_per_node N tools/multiview_bench.py ...                # rays sharded over N GPUs

A synthetic time step: 11 target cameras at 512x288, 7 dynamic + 11 static source views, 64 coarse + 64 fine
samples, chunks of 8192 rays (eval_nvidia.py:305-378 renders each time step from 11 held-out cameras that share
every input but the target camera).

  per-camera  the eval_nvidia.py loop: per camera, the four encoder passes over the 7 + 11 source images
              (coarse and fine encoder, dynamic and static views) and render_single_image_nvi;
  batched     the four encoder passes once, then render_multi_image_nvi over the stacked rays of all cameras.

Under torchrun both forms shard the rays over the ranks (distributed.render_frame_sharded): every rank runs the
encoder on the source images itself, and the pixels (rgb, depth, mask) are gathered on rank 0 -- per camera in
the per-camera form, once per time step in the batched form.

Prints one JSON line on rank 0: rays/s of each form (all cameras' rays over the wall time of the time step,
device-synchronised), the encoder's share of each, whether the two forms' pixels are bit-identical, and the GPU
model and power limit the numbers were measured on.
"""

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def parse():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--cameras", type=int, default=11)
  ap.add_argument("--H", type=int, default=288)
  ap.add_argument("--W", type=int, default=512)
  ap.add_argument("--V-dy", type=int, default=7)
  ap.add_argument("--V-st", type=int, default=11)
  ap.add_argument("--samples", type=int, default=64)
  ap.add_argument("--importance", type=int, default=64)
  ap.add_argument("--chunk", type=int, default=8192)
  ap.add_argument("--reps", type=int, default=2, help="timed time steps per form (after one warm-up step each)")
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
  import torch.distributed as dist
  from dynibar_b200 import distributed as dd, render_ray as rr, sample_ray as sr, synthetic
  from dynibar_b200.feature_network import ResNet
  from dynibar_b200.projection import Projector
  from dynibar_b200.render_image import render_multi_image_nvi, render_single_image_nvi

  rank = int(os.environ.get("RANK", "0"))
  world = int(os.environ.get("WORLD_SIZE", "1"))
  dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
  torch.cuda.set_device(dev)
  if world > 1:
    dist.init_process_group("nccl", device_id=dev)
  rr.set_precision(a.precision)
  H, W, K = a.H, a.W, a.cameras

  # ---- one synthetic time step: shared source views, K target cameras around the rig's target ----
  batch, _, _, frame, t, offs = synthetic.make_scene(H=H, W=W, V_dy=a.V_dy, V_st=a.V_st, rays=1)
  model, args = synthetic.make_model(a.samples, a.importance)
  model = synthetic.model_to(model, dev)
  torch.manual_seed(1)
  model.feature_net = ResNet().to(dev).requires_grad_(False)
  model.feature_net_fine = ResNet().to(dev).requires_grad_(False)
  data = {k: batch[k].to(dev) for k in ("depth_range", "src_rgbs", "src_cameras", "static_src_rgbs",
                                        "static_src_cameras")}
  Kmat = sr.parse_camera(batch["camera"])[2][0]
  samplers = []
  for k in range(K):
    c2w = torch.eye(4)
    c2w[0, 3] = 0.02 * (k - K // 2)
    c2w[1, 3] = 0.005 * ((3 * k) % 5 - 2)
    samplers.append(sr.RaySamplerSingleImage(dict(data, camera=synthetic.camera_vector(H, W, Kmat, c2w)[None]),
                                             dev))
  P = Projector(dev)

  def encode(rb):
    """eval_nvidia.py:331-358: four encoder passes over the dynamic and static source images."""
    src = rb["src_rgbs"].squeeze(0).permute(0, 3, 1, 2)
    st = rb["static_src_rgbs"].squeeze(0).permute(0, 3, 1, 2)
    cb1, _ = model.feature_net(src)
    _, stf = model.feature_net(st)
    cb1f, _ = model.feature_net_fine(src)
    _, stff = model.feature_net_fine(st)
    return (cb1, None, stf), (cb1f, None, stff)

  def render_pixels(fc, ff):
    def fn(local):
      outs = []
      for i in range(0, local["ray_o"].shape[0], a.chunk):
        cb = {k: (v[i:i + a.chunk] if k in ("ray_o", "ray_d", "uv_grid", "camera_index") else v)
              for k, v in local.items()}
        r = rr.render_rays_mv(frame, t, offs, cb, model, P, fc, ff, a.samples, args, inv_uniform=True,
                              N_importance=a.importance, det=True, is_train=False)["outputs_fine_ref"]
        outs.append(torch.cat([r["rgb"], r["depth"][:, None], r["mask"][:, None].float()], 1))
      return torch.cat(outs, 0) if outs else torch.empty(0, 5, device=dev)
    return fn

  def per_camera():
    px = []
    for smp in samplers:
      rb = smp.get_all()
      fc, ff = encode(rb)
      if world == 1:
        r = render_single_image_nvi(frame, t, offs, smp, rb, model, P, a.chunk, a.samples, args, inv_uniform=True,
                                    N_importance=a.importance, det=True, coarse_featmaps=fc, fine_featmaps=ff,
                                    is_train=False)["outputs_fine_ref"]
        px.append(torch.cat([r["rgb"].reshape(-1, 3), r["depth"].reshape(-1, 1), r["mask"].reshape(-1, 1).float()], 1))
      else:
        px.append(dd.render_frame_sharded(render_pixels(fc, ff), rb))
    return px

  def batched():
    rb, counts, _ = sr.stack_ray_batches([smp.get_all() for smp in samplers])
    fc, ff = encode(rb)
    if world == 1:
      rets = render_multi_image_nvi(frame, t, offs, samplers, rb, model, P, a.chunk, a.samples, args,
                                    inv_uniform=True, N_importance=a.importance, det=True, coarse_featmaps=fc,
                                    fine_featmaps=ff, is_train=False)
      return [torch.cat([r["outputs_fine_ref"]["rgb"].reshape(-1, 3), r["outputs_fine_ref"]["depth"].reshape(-1, 1),
                         r["outputs_fine_ref"]["mask"].reshape(-1, 1).float()], 1) for r in rets]
    full = dd.render_frame_sharded(render_pixels(fc, ff), rb)
    return list(full.cpu().split(counts, 0)) if full is not None else None

  def timed(fn, reps):
    times, out = [], None
    for _ in range(reps):
      if world > 1:
        dist.barrier()
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      out = fn()
      torch.cuda.synchronize()
      if world > 1:
        dist.barrier()
      times.append(time.perf_counter() - t0)
    return times, out

  def encoder_time(n_steps):
    rb = samplers[0].get_all()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n_steps):
      encode(rb)
    torch.cuda.synchronize()
    return time.perf_counter() - t0

  # warm-up of every shape the timed steps use, then the two forms alternately
  timed(per_camera, 1)
  timed(batched, 1)
  t_pc, t_b = [], []
  px_pc = px_b = None
  for _ in range(a.reps):
    tt, px_pc = timed(per_camera, 1)
    t_pc += tt
    tt, px_b = timed(batched, 1)
    t_b += tt
  encoder_time(1)
  enc_once = encoder_time(a.reps) / a.reps

  if rank == 0:
    n_rays = K * H * W
    ms_pc, ms_b = 1e3 * min(t_pc), 1e3 * min(t_b)
    same = all(torch.equal(x.cpu(), y.cpu()) for x, y in zip(px_pc, px_b))
    line = {
        "what": "one synthetic time step: %d target cameras at %dx%d, %d dynamic + %d static views, %d+%d samples, "
                "chunk %d, %s" % (K, W, H, a.V_dy, a.V_st, a.samples, a.importance, a.chunk, a.precision),
        "n_gpus": world, "form": "sharded" if world > 1 else "single GPU",
        "per_camera": {"rays_per_s": n_rays / (ms_pc / 1e3), "ms_per_time_step": ms_pc,
                       "ms_all_reps": [1e3 * x for x in t_pc], "encoder_ms": K * 1e3 * enc_once,
                       "encoder_share": K * 1e3 * enc_once / ms_pc},
        "batched": {"rays_per_s": n_rays / (ms_b / 1e3), "ms_per_time_step": ms_b,
                    "ms_all_reps": [1e3 * x for x in t_b], "encoder_ms": 1e3 * enc_once,
                    "encoder_share": 1e3 * enc_once / ms_b},
        "speedup": ms_pc / ms_b, "pixels_bit_identical": same,
        "timing": "wall clock of the whole time step between device synchronisations, best of the reps; "
                  "encoder time measured separately (four passes, synchronised)",
        "gpu": gpu_info(dev.index),
    }
    print(json.dumps(line))
  if world > 1:
    dist.barrier()
    dist.destroy_process_group()
  return 0


if __name__ == "__main__":
  sys.exit(main())
