#!/usr/bin/env python
"""eval_nvidia.py's PSNR / SSIM on one Nvidia-benchmark scene, from the device-resident scene.

  python tools/eval_nvidia.py --scene_path <folder_path>/<scene>/dense --coarse model_coarse.pth --fine model_fine.pth \\
      [--mask_static] [--N_samples 64] [--N_importance 64] [--chunk_size 8192] [--inv_uniform] [--white_bkgd] \\
      [--anti_alias_pooling 1] [--mask_rgb 0] [--occ_weights_mode 0] [--num_basis 6] \\
      [--lpips_alexnet alexnet.pth --lpips_lin alex.pth]

The options are the keys the reference's configs_nvidia/*.txt set that the evaluation reads.  Checkpoints load
through dynibar_b200.model.model_from_checkpoints.  Prints the reference's MOVING lines after every time step and the
AVG lines at the end, in its order.  With --lpips_alexnet (torchvision's AlexNet checkpoint) and --lpips_lin (LPIPS
v0.1's alex.pth) it also computes LPIPS (dynibar_b200.metrics.lpips_views) and prints all nine lines of each block,
as the reference does; without them the LPIPS lines are left out.
"""

import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

LABELS = (("PSNR", 0, 0), ("SSIM", 0, 1), ("DYNAMIC PSNR", 1, 0), ("DYNAMIC SSIM", 1, 1), ("Static PSNR", 2, 0),
          ("Static SSIM", 2, 1))
ROW_NAMES = ("", "DYNAMIC ", "Static ")  # eval_nvidia.py:459-481: per row PSNR, SSIM, LPIPS


def parser():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--scene_path", required=True, help="the reference's <folder_path>/<scene>/dense")
  ap.add_argument("--coarse", required=True, help="coarse checkpoint (the reference's save layout)")
  ap.add_argument("--fine", required=True, help="fine checkpoint")
  ap.add_argument("--mask_static", action="store_true")
  ap.add_argument("--N_samples", type=int, default=64)
  ap.add_argument("--N_importance", type=int, default=64)
  ap.add_argument("--chunk_size", type=int, default=8192)
  ap.add_argument("--inv_uniform", action="store_true")
  ap.add_argument("--white_bkgd", action="store_true")
  ap.add_argument("--anti_alias_pooling", type=int, default=1)
  ap.add_argument("--mask_rgb", type=int, default=0)
  ap.add_argument("--occ_weights_mode", type=int, default=0)
  ap.add_argument("--num_basis", type=int, default=6)
  ap.add_argument("--coarse_feat_dim", type=int, default=32)
  ap.add_argument("--fine_feat_dim", type=int, default=32)
  ap.add_argument("--input_dir", type=int, default=1)
  ap.add_argument("--input_xyz", type=int, default=0)
  ap.add_argument("--device", default="cuda:0")
  ap.add_argument("--lpips_alexnet", default=None, help="torchvision AlexNet checkpoint (with --lpips_lin)")
  ap.add_argument("--lpips_lin", default=None, help="LPIPS v0.1 alex.pth (with --lpips_alexnet)")
  return ap


def print_means(prefix, means, lpips=None):
  if lpips is None:
    for label, r, c in LABELS:
      print("%s %s " % (prefix, label), means[r, c])
    return
  for r, name in enumerate(ROW_NAMES):
    print("%s %sPSNR " % (prefix, name), means[r, 0])
    print("%s %sSSIM " % (prefix, name), means[r, 1])
    print("%s %sLPIPS " % (prefix, name), lpips[r])


def main(argv=None):
  ap = parser()
  args = ap.parse_args(argv)
  if (args.lpips_alexnet is None) != (args.lpips_lin is None):
    ap.error("--lpips_alexnet and --lpips_lin go together")
  args.input_dir, args.input_xyz = bool(args.input_dir), bool(args.input_xyz)
  import torch
  from dynibar_b200 import model as dm
  from dynibar_b200.feature_network import ResNet
  from dynibar_b200.nvidia_scene import NvidiaScene, mean_scores
  from dynibar_b200.projection import Projector
  dev = torch.device(args.device)
  scene = NvidiaScene(args.scene_path, args, dev)
  args.num_frames = scene.num_frames
  print("args.num_frames ", args.num_frames)
  model, info = dm.model_from_checkpoints(args, coarse=args.coarse, fine=args.fine, mono=False, device=dev)
  for k in ("feature_net", "feature_net_fine"):
    enc = ResNet().to(dev)
    enc.load_state_dict(dm._strip(info["encoders"][k]))
    setattr(model, k, enc.eval().requires_grad_(False))
  if args.lpips_alexnet is None:
    res = scene.evaluate(model, Projector(dev), args, on_step=lambda i, s: print_means("MOVING", mean_scores(s)))
    print_means("AVG", res["mean"])
    return res
  from dynibar_b200.metrics import LPIPSWeights
  from dynibar_b200.nvidia_scene import mean_lpips
  w = LPIPSWeights(args.lpips_alexnet, args.lpips_lin, device=dev)
  res = scene.evaluate(model, Projector(dev), args, lpips=w,
                       on_step=lambda i, s, lp: print_means("MOVING", mean_scores(s), mean_lpips(lp)))
  print_means("AVG", res["mean"], res["lpips_mean"])
  return res


if __name__ == "__main__":
  main()
