"""tests/golden/nvi_scene.pt: the reference's Nvidia evaluation front end, run unmodified, on two seeded synthetic
scenes (run where the reference is, as make_golden.py):

    python tests/golden/make_golden_nvi_scene.py

eval_nvidia.py is loaded with runpy, as make_golden_metrics.py loads it, after the modules it imports that cannot run
here are replaced: config (config_parser), imageio (v2.imread / imread through PIL, recording which files are read),
models (PerceptualLoss returning 0), kornia (create_meshgrid, restated) and skimage.* (structural_similarity returns
tests/metrics_ref.ssim_map32).  cv2 is the real one; cv2.resize is wrapped to record its outputs.

1. DynamicVideoDataset items at img_i = 3, one step between and N - 4, for all 12 cameras, collated as the
   DataLoader collates them.  The items of one time step differ only in their target camera (asserted here), so each
   time step keeps the 12 cameras and ground-truth paths, and once: ids, source cameras, depth range, time, which files
   were read, the float stacks by hash and the keys of RaySamplerSingleImage(item).get_all().  The rays of one camera
   of the first time step are kept at every RAY_STRIDE-th pixel.
2. The script's __main__ block with a stand-in renderer that returns nvi_scene_ref.prediction(img_i, camera) (all-zero
   pixels included, so the valid mask matters), Tensor.cuda as the identity, 0 loader workers and the reference's own
   RaySamplerSingleImage on the CPU: the printed per-camera PSNR / SSIM and the MOVING / AVG lines, and every ground
   truth and dynamic mask cv2.resize produced (ground truth by hash, masks bit-packed and compressed).

Scene A: 12 frames of 288 x 8, ground truth at 1080 x 30 (cv2's generic area path in both axes), coloured 3-channel
dynamic masks at 96 x 12 whose channels differ, coarse masks at 300 x 10, mask_static on.
Scene B: 13 frames of 288 x 16 (frames 0 and 12 tie for img_i = 6), ground truth at 576 x 32 and 864 x 48 (integer 2x
and 3x), grey masks at 72 x 20, coarse masks at 144 x 20, mask_static off.  The files are stored as their bytes so the tests can write the scene again; the ground
truth is smooth (a few waves), which keeps its JPEGs small.  tests/nvi_scene_ref.load_golden expands the file
into one record per (time step, camera).
"""

import contextlib
import io
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import metrics_ref as mr  # noqa: E402
import mono_scene_ref as msr  # noqa: E402
import nvi_scene_ref as nsr  # noqa: E402

REF = os.environ.get("DYNIBAR_REFERENCE", "/root/reference")
RAY_STRIDE = 7
SCENES = {
    "A": dict(seed=21, n=12, h=288, w=8, gt_hw=[(1080, 30)], mask_hw=(96, 12), coarse_hw=(300, 10),
              coloured_masks=True, mask_static=True),
    "B": dict(seed=22, n=13, h=288, w=16, gt_hw=[(576, 32), (864, 48)], mask_hw=(72, 20), coarse_hw=(144, 20),
              coloured_masks=False, mask_static=False),
}


def install_stubs(reads):
  from PIL import Image

  def imread(path, **kw):
    reads.append(path)
    return np.asarray(Image.open(path))

  def create_meshgrid(H, W, normalized_coordinates=True):
    assert not normalized_coordinates
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    return torch.stack([xs, ys], -1)[None]

  def structural_similarity(im1, im2, **kw):
    assert kw == dict(multichannel=True, full=True), kw
    S = mr.ssim_map32(im1, im2)
    return float(S[3:-3, 3:-3].mean(dtype=np.float64)), S

  class PerceptualLoss(object):
    def __init__(self, **kw):
      pass

    def forward(self, *a):
      return torch.zeros(())

  mods = {"config": dict(config_parser=None), "imageio": dict(imread=imread), "imageio.v2": dict(imread=imread),
          "models": dict(PerceptualLoss=PerceptualLoss), "kornia": dict(create_meshgrid=create_meshgrid),
          "skimage": {}, "skimage.morphology": {}, "skimage.metrics": dict(structural_similarity=structural_similarity)}
  for name, attrs in mods.items():
    m = types.ModuleType(name)
    for k, v in attrs.items():
      setattr(m, k, v)
    sys.modules[name] = m
  sys.modules["imageio"].v2 = sys.modules["imageio.v2"]
  sys.modules["skimage"].metrics = sys.modules["skimage.metrics"]
  sys.modules["skimage"].morphology = sys.modules["skimage.morphology"]
  sys.path.insert(0, REF)


def scene_files(root):
  out = {}
  for d, _, files in os.walk(root):
    for f in files:
      p = os.path.join(d, f)
      out[os.path.relpath(p, root)] = open(p, "rb").read()
  return out


def main():
  reads, resizes = [], []
  install_stubs(reads)
  import cv2
  from torch.utils.data.dataloader import default_collate
  import torch.utils.data as tud
  from ibrnet import render_image, sample_ray
  import ibrnet.model

  real_resize = cv2.resize

  def resize(src, dsize, **kw):
    out = real_resize(src, dsize, **kw)
    resizes.append((kw.get("interpolation"), src.shape, out))
    return out

  cv2.resize = resize
  g = runpy.run_path(os.path.join(REF, "eval_nvidia.py"), run_name="eval_nvidia_golden")
  Dataset = g["DynamicVideoDataset"]
  out = dict(scenes={})
  with tempfile.TemporaryDirectory() as tmp:
    for name, sc in SCENES.items():
      s = nsr.synthetic_scene(sc["seed"], sc["n"], sc["h"], sc["w"], sc["gt_hw"], sc["mask_hw"], sc["coarse_hw"],
                              sc["coloured_masks"])
      root = nsr.write_scene(os.path.join(tmp, name, "dense"), s)
      n = sc["n"]
      for t in list(range(n)):  # only the ground truth and masks the evaluation reads are kept
        for c in range(nsr.CYCLE):
          if not (3 <= t < n - 3) or c == t % nsr.CYCLE:
            os.remove(os.path.join(root, "mv_images", "%05d" % t, "cam%02d.jpg" % (c + 1)))
            os.remove(os.path.join(root, "mv_masks", "%05d" % t, "cam%02d.png" % (c + 1)))
      args = types.SimpleNamespace(folder_path=tmp, mask_static=sc["mask_static"], eval_scenes=[name])
      rec = dict(files=scene_files(root), mask_static=sc["mask_static"], n=n, steps={})
      ds0 = Dataset(0, args, scenes=[name])
      rec.update(c2w=torch.from_numpy(ds0.train_poses), K=torch.from_numpy(ds0.train_intrinsics),
                 depth_range=torch.tensor(ds0.render_depth_range[0]), hw=(ds0.h[0], ds0.w[0]))
      for img_i in (3, (3 + n - 4) // 2, n - 4):
        ds = Dataset(img_i, args, scenes=[name])
        cams, paths, step = [], [], None
        for cam in range(len(ds)):
          del reads[:]
          data = default_collate([ds[cam]])
          item = dict(reads=[os.path.relpath(r, root) for r in reads])
          for k in ("src_cameras", "static_src_cameras", "depth_range", "ref_time", "id", "nearest_pose_ids"):
            item[k] = data[k]
          item["hash"] = {k: msr.hash_f32(data[k]) for k in ("src_rgbs", "static_src_rgbs", "static_src_masks")}
          item["dtypes"] = {k: (str(v.dtype), tuple(v.shape)) for k, v in data.items() if torch.is_tensor(v)}
          rb = sample_ray.RaySamplerSingleImage(data, device="cpu").get_all()
          item["ray_keys"] = {k: None if v is None else (str(v.dtype), tuple(v.shape)) for k, v in rb.items()}
          if step is None:
            step = item
            if not rec["steps"]:  # the reference's own rays of one camera, at every RAY_STRIDE-th pixel
              sel = torch.arange(0, rb["ray_o"].shape[0], RAY_STRIDE)
              step["rays"] = dict({k: rb[k][sel] for k in ("ray_o", "ray_d", "uv_grid")}, sel=sel, cam=cam)
          else:  # the items of one time step differ only in their target camera
            assert all(torch.equal(item[k], step[k]) if torch.is_tensor(item[k]) else item[k] == step[k]
                       for k in item), (name, img_i, cam)
          cams.append(data["camera"][0])
          paths.append(os.path.relpath(data["rgb_path"][0], root))
        step.update(camera=torch.stack(cams), rgb_path=paths)
        rec["steps"][img_i] = step
      out["scenes"][name] = rec

      # the __main__ block
      def render(frame_idx, time_embedding, time_offset, ray_sampler, ray_batch, **kw):
        cam = int(os.path.basename(ray_sampler.rgb_path[0])[3:5]) - 1
        pred = nsr.prediction(frame_idx[0], cam, ray_sampler.H, ray_sampler.W)
        return dict(outputs_fine_ref=dict(rgb=torch.from_numpy(pred), depth=torch.zeros(pred.shape[:2])))

      class Model(object):
        def __init__(self, *a, **kw):
          self.feature_net = self.feature_net_fine = lambda x: (x, x)

        def switch_to_eval(self):
          pass

      class Loader(tud.DataLoader):
        def __init__(self, ds, **kw):
          kw["num_workers"] = 0
          super().__init__(ds, **kw)

      class Sampler(sample_ray.RaySamplerSingleImage):
        def __init__(self, data, device, **kw):
          super().__init__(data, "cpu", **kw)

      cli = types.SimpleNamespace(folder_path=tmp, eval_scenes=[name], mask_static=sc["mask_static"],
                                  eval_dataset="Nvidia", expname="golden", chunk_size=4096, N_samples=64,
                                  inv_uniform=True, N_importance=0, white_bkgd=False)
      sys.modules["config"].config_parser = lambda: types.SimpleNamespace(parse_args=lambda: cli)
      saved = (ibrnet.model.DynibarFF, render_image.render_single_image_nvi, tud.DataLoader,
               sample_ray.RaySamplerSingleImage, torch.Tensor.cuda)
      ibrnet.model.DynibarFF, render_image.render_single_image_nvi, tud.DataLoader = Model, render, Loader
      sample_ray.RaySamplerSingleImage, torch.Tensor.cuda = Sampler, lambda self, *a, **k: self
      del resizes[:]
      buf = io.StringIO()
      try:
        with contextlib.redirect_stdout(buf):
          runpy.run_path(os.path.join(REF, "eval_nvidia.py"), run_name="__main__")
      finally:
        (ibrnet.model.DynibarFF, render_image.render_single_image_nvi, tud.DataLoader,
         sample_ray.RaySamplerSingleImage, torch.Tensor.cuda) = saved
      rec["printed"] = buf.getvalue()
      gt, masks = [], []
      for interp, shape, o in resizes:
        if interp == cv2.INTER_AREA:
          gt.append(msr.hash_f32(np.float32(o) / 255))
        elif interp == cv2.INTER_NEAREST and len(shape) == 3:
          masks.append(o)
      rec["gt_hash"], rec["dynamic_masks"] = gt, nsr.pack_masks(masks)
  path = os.path.join(HERE, "nvi_scene.pt")
  torch.save(msr.to_numpy(out), path, pickle_protocol=4)
  print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
  main()
