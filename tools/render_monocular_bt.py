#!/usr/bin/env python
"""render_monocular_bt.py's bullet-time video of a trained monocular model, from the device-resident scene.

  python tools/render_monocular_bt.py --scene_path <folder_path>/<scene>/dense --coarse model.pth --render_idx 20 \\
      [--out .] [--eval_dataset Kid-Running] [--expname exp] [--training_height 288] [--num_source_views 7] \\
      [--max_range 10] [--num_vv 3] [--mask_src_view] [--N_samples 64] [--chunk_size 8192] [--inv_uniform] \\
      [--anti_alias_pooling 1] [--mask_rgb 1] [--occ_weights_mode 0]

The options are the keys of the reference's configs (configs/test_*.txt) that the script reads.  The checkpoint loads
through dynibar_b200.model.model_from_checkpoints (mono=True).  Writes rgb_out/{i}.png under
<out>/<eval_dataset>/<expname>/<render_idx>/<scene>_<step:06d>/videos/, as the script does (RGB PNGs, cropped by 3 %),
and prints the wall time split into load, encoder, render and write.  A render_idx >= 0 renders the bullet-time sweep
of that frame, i = 0..49; a negative render_idx renders the stabilised video of the n frames, camera i at frame i's
time, i = 3..n-4 (each camera needs the frames i-3 .. i+3).
"""

import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def parser():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--scene_path", required=True, help="the reference's <folder_path>/<scene>/dense")
  ap.add_argument("--coarse", required=True, help="DynibarMono checkpoint (the reference's save layout)")
  ap.add_argument("--render_idx", type=int, required=True)
  ap.add_argument("--out", default=".", help="directory the reference's relative output path starts from")
  ap.add_argument("--eval_dataset", default="Nvidia")
  ap.add_argument("--expname", default="exp")
  ap.add_argument("--training_height", type=int, default=288)
  ap.add_argument("--num_source_views", type=int, default=7)
  ap.add_argument("--max_range", type=int, default=10)
  ap.add_argument("--num_vv", type=int, default=3)
  ap.add_argument("--mask_src_view", action="store_true")
  ap.add_argument("--N_samples", type=int, default=64)
  ap.add_argument("--N_importance", type=int, default=0)
  ap.add_argument("--chunk_size", type=int, default=8192)
  ap.add_argument("--inv_uniform", action="store_true")
  ap.add_argument("--white_bkgd", action="store_true")
  ap.add_argument("--anti_alias_pooling", type=int, default=1)
  ap.add_argument("--mask_rgb", type=int, default=1)
  ap.add_argument("--occ_weights_mode", type=int, default=0)
  ap.add_argument("--num_basis", type=int, default=6)
  ap.add_argument("--coarse_feat_dim", type=int, default=32)
  ap.add_argument("--fine_feat_dim", type=int, default=32)
  ap.add_argument("--input_dir", type=int, default=1)
  ap.add_argument("--input_xyz", type=int, default=0)
  ap.add_argument("--device", default="cuda:0")
  return ap


def main(argv=None):
  args = parser().parse_args(argv)
  args.input_dir, args.input_xyz = bool(args.input_dir), bool(args.input_xyz)
  import cv2
  import torch
  from dynibar_b200 import model as dm
  from dynibar_b200.bt_scene import BulletTimeScene
  from dynibar_b200.feature_network import ResNet
  from dynibar_b200.projection import Projector
  dev = torch.device(args.device)

  def now():
    torch.cuda.synchronize(dev)
    return time.perf_counter()

  t0 = now()
  scene = BulletTimeScene(args.scene_path, args, dev)
  args.num_frames = scene.num_frames
  t_load = now() - t0
  model, info = dm.model_from_checkpoints(args, coarse=args.coarse, mono=True, device=dev)
  for k in ("feature_net", "feature_net_st"):
    enc = ResNet().to(dev)
    enc.load_state_dict(dm._strip(info["encoders"][k]))
    setattr(model, k, enc.eval().requires_grad_(False))
  scene_name = os.path.basename(os.path.dirname(os.path.normpath(args.scene_path)))
  out_dir = os.path.join(args.out, args.eval_dataset, args.expname, str(args.render_idx),
                         "%s_%06d" % (scene_name, info.get("coarse_step", 0)), "videos")
  os.makedirs(os.path.join(out_dir, "rgb_out"), exist_ok=True)
  print("saving results to {}".format(out_dir))
  projector = Projector(dev)
  t = dict(encoder=0.0, render=0.0, write=0.0)
  t_sweep = now()
  for g in range(len(scene)):
    step = scene.group_batch(g)
    with torch.no_grad():
      t1 = now()
      feats = scene.encode(step, model)
      t2 = now()
      rgb = scene.render(step, feats, model, projector, args)
      frames = scene.frames_device(rgb).cpu().numpy()
      t3 = now()
    for i, f in zip(step["cameras"], frames):
      cv2.imwrite(os.path.join(out_dir, "rgb_out", "{}.png".format(i)), f[:, :, ::-1])  # RGB, as imageio writes
    t4 = now()
    t["encoder"] += t2 - t1
    t["render"] += t3 - t2
    t["write"] += t4 - t3
  total = now() - t_sweep
  what = ("stabilised video of %d frames" % scene.num_frames if scene.stabilized
          else "bullet-time sweep of frame %d" % args.render_idx)
  print("%s: %d cameras in %d groups; load %.3f s, sweep %.3f s (encoder %.3f s, render %.3f s, write %.3f s)"
        % (what, sum(hi - lo for lo, hi in scene.groups), len(scene), t_load, total, t["encoder"], t["render"],
           t["write"]))
  return out_dir


if __name__ == "__main__":
  main()
