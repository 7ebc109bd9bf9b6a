"""Writes a monocular scene's virtual source views, the files training and rendering read when num_vv > 0:

  <data_dir>/dense/source_vv_poses.npy                          [8, 3, 4, N] float32
  <data_dir>/dense/source_virtual_views_<W>x<H>/%05d/%02d.png    8 views per frame, H = 288

  python tools/make_virtual_views.py --data_dir <scene> --cvd_dir <dynamic-video-depth output with %05d.npz>

A replacement for the reference's render_source_vv.py: the same inputs and outputs, with the splat, the Sobel alpha
and the masking on the GPU (dynibar_b200.virtual_views) instead of the external `splatting` extension, kornia and
skimage.  Resizing stays on the host with cv2, as in the reference.
"""

import argparse
import glob
import os
import sys

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dynibar_b200 import virtual_views as vv  # noqa: E402


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--data_dir", required=True, help="scene directory (holds dense/images/00000.png or .jpg)")
  ap.add_argument("--cvd_dir", required=True, help="video depth directory: one .npz per frame")
  ap.add_argument("--device", default="cuda:0")
  args = ap.parse_args()
  dev = torch.device(args.device)

  data_path = os.path.join(args.data_dir, "dense")
  npz_paths = sorted(glob.glob(os.path.join(args.cvd_dir, "*.npz")))
  if not npz_paths:
    raise SystemExit("make_virtual_views: no .npz in %s" % args.cvd_dir)
  first = os.path.join(data_path, "images", "00000.png")
  if not os.path.exists(first):
    first = os.path.join(data_path, "images", "00000.jpg")
  o_img = cv2.imread(first, cv2.IMREAD_UNCHANGED)
  if o_img is None:
    raise SystemExit("make_virtual_views: cannot read %s" % first)
  final_h = vv.FINAL_H
  final_w = int(round(final_h * float(o_img.shape[1]) / float(o_img.shape[0])))
  save_dir = os.path.join(data_path, "source_virtual_views_%dx%d" % (final_w, final_h))
  os.makedirs(save_dir, exist_ok=True)

  frames = [dict(np.load(p)) for p in npz_paths]
  Ks = [vv.scaled_intrinsics(f["K"], f["img_1"].shape[2:], (final_h, final_w)) for f in frames]
  npy, tgt_c2w = vv.virtual_view_poses(np.stack([f["cam_c2w"][0] for f in frames]),
                                       [f["depth"][0, 0] for f in frames], Ks[-1], (final_h, final_w))
  np.save(os.path.join(data_path, "source_vv_poses.npy"), npy)

  for i, (f, K) in enumerate(zip(frames, Ks)):
    if abs(K[0, 0] - K[1, 1]) / abs(K[0, 0] + K[1, 1]) >= 0.005:
      raise SystemExit("make_virtual_views: frame %d has fx %g != fy %g" % (i, K[0, 0], K[1, 1]))
    img = cv2.resize(f["img_1"][0].transpose(1, 2, 0), (final_w, final_h), interpolation=cv2.INTER_AREA)
    disp = cv2.resize(1.0 / f["depth"][0, 0], (final_w, final_h), interpolation=cv2.INTER_LINEAR)
    views = vv.render_virtual_views(torch.from_numpy(np.ascontiguousarray(img, np.float32)).to(dev),
                                    torch.from_numpy(np.ascontiguousarray(disp, np.float32)).to(dev),
                                    K, f["cam_c2w"][0], tgt_c2w[i]).cpu().numpy()
    sub = os.path.join(save_dir, "%05d" % i)
    os.makedirs(sub, exist_ok=True)
    for k, v in enumerate(views):
      cv2.imwrite(os.path.join(sub, "%02d.png" % k), np.ascontiguousarray(v[..., ::-1]))  # RGB -> cv2's BGR
    print(sub)


if __name__ == "__main__":
  main()
