"""tests/golden/mono_scene.pt: the reference's monocular training loader, run unmodified, on two seeded synthetic scenes
(run where the reference is, as make_golden.py):

    python tests/golden/make_golden_scene.py

ibrnet/data_loaders/monocular.py (MonocularDataset) and ibrnet/sample_ray.py (RaySamplerSingleImage) are imported
as they are, after three modules they import that cannot run here are replaced:
  imageio    imread reads through PIL, as imageio 2.22 does for PNG;
  skimage    morphology.disk / erosion as skimage 0.19.3 computes them (tests/mono_scene_ref.py: scipy grey_erosion,
             disk footprint, mode 'reflect');
  kornia     create_meshgrid(H, W, normalized_coordinates=False), restated.
load_src_view is wrapped to record which file (and which mask) each view came from.

Tensors are stored as numpy arrays (tests/mono_scene_ref.load_golden turns them back).  The raw arrays are stored
compressed (compressible() keeps few distinct values); the items keep ids, cameras, masks
(bit-packed) and rays in full and the float images, disparity and flows by hash.

Scene A: 16 frames of 288 x 4 (images_4x288), masks at frame size: the motion mask is eroded at frame size.
Scene B: training_height 24, 16 frames of 24 x 40, 3-channel dynamic masks and static masks at 30 x 50: every resize
is non-trivial and the erosion runs at 288 x 480.
num_source_views 3, max_range 9, num_vv 3, init_decay_epoch 2.  Items at several seeds and epochs on both sides of
init_decay_epoch, a seed whose 0.5 % draw adds the target frame to the anchor views, mask_src_view on and off and
erosion_radius 0, 1, 3 and 5.
"""

import io
import os
import sys
import tempfile
import types

import numpy as np
import scipy.ndimage as ndi
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import mono_scene_ref as msr  # noqa: E402

REF = os.environ.get("DYNIBAR_REFERENCE", "/root/reference")
N_RAND = 32
SCENES = {
    "A": dict(seed=11, n=16, h=288, w=4, height=288, mask_hw=None, orig_hw=(576, 8), mask_channels=0, far_max=6.0),
    "B": dict(seed=12, n=16, h=24, w=40, height=24, mask_hw=(30, 50), orig_hw=(48, 80), mask_channels=3,
              far_max=40.0),
}
BASE = dict(num_source_views=3, max_range=9, num_vv=3, init_decay_epoch=2)
# (scene, mask_src_view, erosion_radius, [(seed, epoch, pixel_seed, sample_mode)])
CASES = [
    ("A", True, 3, [(0, 0, 100, "center"), (1, 3, 101, "uniform"), (2, 6, 102, "center")]),
    ("A", False, 0, [(3, 1, 103, "center"), (4, 4, 104, "uniform")]),
    ("A", True, 5, [(5, 2, 105, "uniform")]),
    ("B", True, 1, [(6, 0, 106, "center"), (7, 2, 107, "uniform"), (8, 5, 108, "center")]),
    ("B", False, 3, [(9, 1, 109, "uniform")]),
    ("B", True, 5, [(10, 7, 110, "center")]),
    ("B", True, 0, [(11, 3, 111, "uniform")]),
]


def install_stubs():
  def create_meshgrid(H, W, normalized_coordinates=True):
    assert not normalized_coordinates
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    return torch.stack([xs, ys], -1)[None]

  mods = {
      "imageio": dict(imread=msr.imread),
      "skimage": {}, "skimage.morphology": dict(disk=msr.disk,
                                                 erosion=lambda image, fp: ndi.grey_erosion(image, footprint=fp)),
      "kornia": dict(create_meshgrid=create_meshgrid),
  }
  for name, attrs in mods.items():
    m = types.ModuleType(name)
    for k, v in attrs.items():
      setattr(m, k, v)
    sys.modules[name] = m
  sys.modules["skimage"].morphology = sys.modules["skimage.morphology"]
  sys.path.insert(0, REF)


def find_rare_seed(n, cfg, epoch):
  """A seed whose 0.5 % draw (the third call of __getitem__) includes the target frame in the anchor views."""
  for seed in range(20000):
    rs = np.random.RandomState(seed)
    rs.randint(3, n - 3)
    max_step = min(3, epoch // cfg["init_decay_epoch"] + 1)
    rs.choice(2 * max_step)
    if rs.choice([0, 1], p=[1.0 - 0.005, 0.005]):
      return seed
  raise RuntimeError("no seed")


def compressible(s):
  """Fewer distinct values where the tests do not need them, so the stored raw arrays compress: frames take four
  colour values, virtual views two (grey), disparity eight, flows three (mostly 0); flows and flow masks are zero on
  the frames __getitem__ never draws (0-2, n-3..)."""
  s = dict(s)
  s["frames"] = (s["frames"] // 64 * 85).astype(np.uint8)
  s["vviews"] = np.repeat(np.where(s["vviews"][..., :1] >= 128, 170, 85), 3, -1).astype(np.uint8)
  s["flows"] = (np.sign(s["flows"]) * (np.abs(s["flows"]) > 1.0) * 0.75).astype(np.float32)
  s["disp"] = (np.ceil(s["disp"] * 4) / 4).astype(np.float32)
  n = len(s["frames"])
  for k in ("flows", "flow_masks"):
    s[k] = s[k].copy()
    s[k][:3] = 0
    s[k][n - 3:] = 0
  return s


def npz_bytes(d):
  buf = io.BytesIO()
  np.savez_compressed(buf, **d)
  return buf.getvalue()


def main():
  install_stubs()
  from ibrnet.data_loaders import monocular
  from ibrnet import sample_ray
  from torch.utils.data.dataloader import default_collate

  rare = find_rare_seed(16, BASE, 4)
  CASES.append(("A", True, 1, [(rare, 4, 112, "center")]))
  out = dict(scenes={}, cases=[], base=dict(BASE), n_rand=N_RAND, rare_seed=rare)
  with tempfile.TemporaryDirectory() as tmp:
    raw = {}
    for name, sc in SCENES.items():
      s = msr.synthetic_scene(sc["seed"], sc["n"], sc["h"], sc["w"], sc["mask_hw"], sc["orig_hw"],
                              sc["mask_channels"], sc["far_max"])
      s = compressible(s)
      raw[name] = s
      msr.write_scene(os.path.join(tmp, name, "dense"), s)
      out["scenes"][name] = dict(raw=npz_bytes(s), height=sc["height"])
    rec = []
    load = monocular.MonocularDataset.load_src_view

    def load_src_view(self, rgb_file, pose, intrinsics, st_mask_path=None):
      rec.append((os.path.relpath(rgb_file, self.scene_path),
                  None if st_mask_path is None else os.path.relpath(st_mask_path, self.scene_path)))
      return load(self, rgb_file, pose, intrinsics, st_mask_path)

    monocular.MonocularDataset.load_src_view = load_src_view
    for name, msv, radius, items in CASES:
      args = types.SimpleNamespace(folder_path=tmp, training_height=SCENES[name]["height"], mask_src_view=msv,
                                   erosion_radius=radius, **BASE)
      ds = monocular.MonocularDataset(args, "train", scenes=(name,))
      sc = out["scenes"][name]
      if "c2w" not in sc:
        sc.update(c2w=torch.from_numpy(ds.train_poses), K=torch.from_numpy(ds.train_intrinsics),
                  vv_c2w=torch.from_numpy(ds.src_vv_c2w_mats), scale=np.float64(ds.scale),
                  scale_dtype=str(np.asarray(ds.scale).dtype),
                  depth_range=torch.tensor(ds.train_depth_range[0], dtype=torch.float64),
                  rgb_files=[os.path.relpath(f, ds.scene_path) for f in ds.train_rgb_files])
      for seed, epoch, pix_seed, mode in items:
        ds.set_epoch(epoch)
        np.random.seed(seed)
        del rec[:]
        item = ds[0]
        data = default_collate([item])
        sample_ray.rng = np.random.RandomState(pix_seed)
        rb = sample_ray.RaySamplerSingleImage(data, torch.device("cpu")).random_sample(N_RAND, mode)
        c = dict(scene=name, mask_src_view=msv, erosion_radius=radius, seed=seed, epoch=epoch, pixel_seed=pix_seed,
                 sample_mode=mode, loads=list(rec), rgb_path=os.path.relpath(data["rgb_path"][0], ds.scene_path))
        for k in ("id", "anchor_id", "num_frames", "ref_time", "anchor_time", "nearest_pose_ids",
                  "anchor_nearest_pose_ids", "camera", "anchor_camera", "src_cameras", "static_src_cameras",
                  "anchor_src_cameras", "depth_range"):
          c[k] = data[k]
        for k in ("motion_mask", "static_mask"):
          assert torch.equal(data[k], data[k].bool().float())
          c[k] = msr.pack_mask(data[k][0])
        c["hash"] = {k: msr.hash_f32(data[k]) for k in ("rgb", "disp", "flows", "masks", "src_rgbs",
                                                         "static_src_rgbs", "anchor_src_rgbs")}
        c["dtypes"] = {k: (str(v.dtype), tuple(v.shape)) for k, v in data.items() if torch.is_tensor(v)}
        c["rays"] = {k: v for k, v in rb.items() if torch.is_tensor(v) and k in (
            "ray_o", "ray_d", "rgb", "disp", "motion_mask", "static_mask", "uv_grid", "flows", "masks")}
        c["rays"]["selected_inds"] = torch.from_numpy(np.asarray(rb["selected_inds"]))
        c["ray_keys"] = sorted(rb)
        out["cases"].append(c)
  assert any(int(c["id"]) in c["anchor_nearest_pose_ids"][0].tolist() for c in out["cases"])
  path = os.path.join(HERE, "mono_scene.pt")
  # numpy arrays pickle inline (far smaller than one zip record per tensor); protocol 4 stores bytes as they are
  torch.save(msr.to_numpy(out), path, pickle_protocol=4)
  print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
  main()
