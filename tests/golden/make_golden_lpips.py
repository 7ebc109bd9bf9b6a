"""tests/golden/lpips_glue.pt: eval_nvidia.py's LPIPS glue, run unmodified on a seeded synthetic scene wide enough for
AlexNet (run where the reference is, as make_golden.py):

    python tests/golden/make_golden_lpips.py

The script runs as make_golden_nvi_scene.py runs it (its stubs, a stand-in renderer returning
nvi_scene_ref.prediction, 0 loader workers), except that models.PerceptualLoss evaluates tests/lpips_ref.lpips in
PLAIN mode with lpips_ref.random_weights(WEIGHTS_SEED) on exactly the tensors the script passes (im2tensor's images in
[-1, 1] and its [1, 3, H, W] masks), and returns a one-element tensor.  This pins the glue: which images, which mask
rows, im2tensor and the argument order.  Scenes A and B of nvi_scene.pt are 8 and 16 px wide, too narrow for AlexNet
(the real PerceptualLoss would fail on them as well).

Scene C: 12 frames of 288 x 32, ground truth at 576 x 64, grey masks at 72 x 40, coarse masks at 144 x 40,
mask_static off.  Stored: the scene's files, the printed per-camera LPIPS values {(img_i, camera): [3]} and the
AVG LPIPS lines [3] (full, DYNAMIC, Static).
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
sys.path.insert(0, HERE)
import lpips_ref as lr  # noqa: E402
import make_golden_nvi_scene as mg  # noqa: E402
import nvi_scene_ref as nsr  # noqa: E402

WEIGHTS_SEED = 5
SCENE = dict(seed=23, n=12, h=288, w=32, gt_hw=[(576, 64)], mask_hw=(72, 40), coarse_hw=(144, 40),
             coloured_masks=False, mask_static=False)


def printed_lpips(text):
  """eval_nvidia.py's stdout -> ({(img_i, cam): float64 [3]} of the third value of its three per-camera lines,
  [3] of the AVG LPIPS lines)."""
  per, avg, cur, rows = {}, {}, None, []
  for line in text.splitlines():
    f = line.split()
    if line.startswith("img_i "):
      cur, rows = (int(f[1]), int(f[2])), []
    elif line.startswith("AVG"):
      avg[" ".join(f[:-1])] = float(f[-1])
    elif cur is not None and len(f) == 3 and len(rows) < 3 and not line.startswith("MOVING"):
      rows.append(float(f[2]))
      if len(rows) == 3:
        per[cur] = np.array(rows)
  return per, np.array([avg["AVG LPIPS"], avg["AVG DYNAMIC LPIPS"], avg["AVG Static LPIPS"]])


def main():
  reads = []
  mg.install_stubs(reads)
  alex, lin = lr.random_weights(WEIGHTS_SEED)

  class PerceptualLoss(object):
    def __init__(self, **kw):
      assert kw == dict(model="net-lin", net="alex", use_gpu=True, version=0.1), kw

    def forward(self, in0, in1, mask):
      cl = lambda t: t.permute(0, 2, 3, 1).numpy()
      return lr.lpips(cl(in0), cl(in1), cl(mask), alex, lin, mode="plain")[:, 0].float()

  sys.modules["models"].PerceptualLoss = PerceptualLoss
  import torch.utils.data as tud
  from ibrnet import render_image, sample_ray
  import ibrnet.model

  sc = SCENE
  with tempfile.TemporaryDirectory() as tmp:
    name = "C"
    s = nsr.synthetic_scene(sc["seed"], sc["n"], sc["h"], sc["w"], sc["gt_hw"], sc["mask_hw"], sc["coarse_hw"],
                            sc["coloured_masks"])
    root = nsr.write_scene(os.path.join(tmp, name, "dense"), s)
    n = sc["n"]
    for t in range(n):  # only the ground truth and masks the evaluation reads are kept
      for c in range(nsr.CYCLE):
        if not (3 <= t < n - 3) or c == t % nsr.CYCLE:
          os.remove(os.path.join(root, "mv_images", "%05d" % t, "cam%02d.jpg" % (c + 1)))
          os.remove(os.path.join(root, "mv_masks", "%05d" % t, "cam%02d.png" % (c + 1)))
    files = mg.scene_files(root)

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
    buf = io.StringIO()
    try:
      with contextlib.redirect_stdout(buf):
        runpy.run_path(os.path.join(mg.REF, "eval_nvidia.py"), run_name="__main__")
    finally:
      (ibrnet.model.DynibarFF, render_image.render_single_image_nvi, tud.DataLoader,
       sample_ray.RaySamplerSingleImage, torch.Tensor.cuda) = saved
  per, avg = printed_lpips(buf.getvalue())
  assert len(per) == (n - 6) * (nsr.CYCLE - 1), len(per)
  out = dict(files=files, mask_static=sc["mask_static"], weights_seed=WEIGHTS_SEED, per_camera=per, avg=avg)
  path = os.path.join(HERE, "lpips_glue.pt")
  torch.save(out, path, pickle_protocol=4)
  print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
  main()
