"""tests/golden/bt_stab.pt: what the reference's render_monocular_bt.py loader gives for the stabilised video
(render_idx < 0) on small on-disk scenes, run where the reference is:

    python tests/golden/make_golden_bt_stab.py

Two seeded 16-frame scenes at 48x36, with the virtual views of every frame, are written to a temporary `dense` folder
by make_golden_bt_scene.py's scene builder and writer, with its stubs (imageio as a cv2 reader; empty model, renderer
and config modules).  load_mono_data(render_idx=-1) and the script's DynamicVideoDataset run unmodified over them.
Two adjustments, both outside the reference's code:
  - __getitem__ reads every time-dependent value (the temporal views, the static views' distance test, the virtual
    views' folder and poses, ref_time and id) from the fixed self.render_idx, so with render_idx = -1 every camera
    would render at time -1/n from wrapped-around frames.  Camera i of the stabilised path is recorded as
    __getitem__(i) returns it after `dataset.render_idx = i`, for i = 3..12 (each needs frames i-3 .. i+3).
  - numpy 1.x, the reference's environment, computes the depth range in float64 (`np.max(bds) + 15.0` and
    `x * 0.9` on float32 scalars); numpy 2 keeps float32.  The constructor's render_depth_range is recomputed from
    the same bounds as numpy 1.x evaluates it, as make_golden_bt_scene.py does.

Recorded per case: load_mono_data's render_poses [16, 3, 5], and per camera i: camera, src_cameras,
static_src_cameras, depth_range, ref_time, id, nearest_pose_ids and the selection (temporal, virtual-view and static
ids, from the files read), and the SHA-256 of the camera's src_rgbs / static_src_rgbs.  The source cameras are stored
as distinct rows and per-slot indices.  The scenes are stored as their seeds and a SHA-256 of their arrays
(tests/bt_stab_ref.py rebuilds them), which keeps the file small: their 128 virtual views alone are 650 KB.
"""

import os
import re
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import bt_scene_ref as bsr  # noqa: E402
import bt_stab_ref as bst  # noqa: E402
import make_golden_bt_scene as mgb  # noqa: E402

REF = os.environ.get("DYNIBAR_REFERENCE", "/root/reference")
# scene -> (seed, largest bound, mask shape): C's 3-channel masks at 40x30; D's largest bound is below 10, where
# training's far rule differs
SCENES = {"C": (5, 30.0, (30, 40, 3)), "D": (6, 6.0, (18, 24))}
# (scene, mask_src_view, num_source_views, max_range, num_vv).  max_range 6 with 3 views takes every second frame;
# within 7.5 frames of camera 3 or 12 fewer than 7 remain, so the [::5] fallback fills in.
CASES = (("C", True, 3, 6, 3), ("D", False, 3, 6, 2))


def main():
  sys.path.insert(0, REF)
  reads = []
  mgb._install_stubs(reads)
  from ibrnet.data_loaders import llff_data_utils as llff
  import render_monocular_bt as bt
  scenes = {name: bst.make_scene(*r) for name, r in SCENES.items()}
  cases = []
  with tempfile.TemporaryDirectory() as tmp:
    for name, s in scenes.items():
      bsr.write_scene(os.path.join(tmp, name, "dense"), s)
    for name, mask, nsv, max_range, num_vv in CASES:
      args = types.SimpleNamespace(folder_path=tmp, num_source_views=nsv, mask_src_view=mask, render_idx=-1,
                                   max_range=max_range, num_vv=num_vv, training_height=bsr.SCENE_H)
      bt.args = args  # __getitem__ reads the script's global args
      ds = bt.DynamicVideoDataset(args, scenes=[name])
      _, _, _, bds, render_poses, _, files, _ = llff.load_mono_data(os.path.join(tmp, name, "dense"),
                                                                    height=bsr.SCENE_H, render_idx=-1,
                                                                    load_imgs=False)
      assert len(ds) == len(files) == bsr.N_FRAMES and render_poses.dtype == np.float32
      # numpy 1.x's depth range (the module docstring)
      near, top = np.float64(np.min(bds)), np.float64(np.max(bds))
      far = min(50, top + 15.0) if top < 10 else min(50, max(20, top))
      ds.render_depth_range = [[near, np.float64(far)]] * ds.num_frames
      rec = dict(scene=name, mask_src_view=mask, render_idx=-1, num_source_views=nsv, max_range=max_range,
                 num_vv=num_vv, render_poses=torch.from_numpy(render_poses), ids=[], camera=[], src_cameras=[],
                 static_src_cameras=[], selections=[], ref_time=[], images={})
      for i in range(bst.FIRST, bst.LAST + 1):
        ds.render_idx = i  # the one adjustment (the module docstring)
        del reads[:]
        item = ds[i]
        paths = reads[1:]  # reads[0]: the unused ground truth
        frame_of = lambda p: int(re.search(r"(\d+)\.png$", p).group(1))
        temporal = [frame_of(p) for p in paths[:7]]
        vv = [frame_of(p) for p in paths[7:7 + num_vv]]
        assert all(os.path.join("source_virtual_views_%dx%d" % (bsr.SCENE_W, bsr.SCENE_H), "%05d" % i) in p
                   for p in paths[7:7 + num_vv])
        rest = paths[7 + num_vv:]
        static = [frame_of(p) for p in rest if "images_" in p]
        assert len(rest) == len(static) * (2 if mask else 1), rest
        assert list(item["nearest_pose_ids"]) == temporal == list(range(i - 3, i + 4))
        assert item["id"] == i
        rec["ids"].append(i)
        rec["selections"].append((temporal, vv, static))
        rec["camera"].append(item["camera"])
        rec["src_cameras"].append(item["src_cameras"])
        rec["static_src_cameras"].append(item["static_src_cameras"])
        rec["ref_time"].append(item["ref_time"])
        assert item["depth_range"].dtype == torch.float64
        if i == bst.FIRST:
          rec["depth_range"] = item["depth_range"]
        assert torch.equal(item["depth_range"], rec["depth_range"])
        rec["images"][i] = (bsr.digest(item["src_rgbs"]), bsr.digest(item["static_src_rgbs"]))
      rec["camera"] = torch.stack(rec["camera"])
      mgb._pack_cameras(rec, torch.stack(rec.pop("src_cameras")), torch.stack(rec.pop("static_src_cameras")))
      # a static frame off the interval grid or outside the distance test came from the [::5] fallback
      rec["fallback"] = [any(f % (max_range // nsv) or abs(f - i) > max_range + nsv * 0.5 for f in sel[2])
                         for i, sel in zip(rec["ids"], rec["selections"])]
      cases.append(rec)
  assert all(c["fallback"][0] and c["fallback"][-1] for c in cases)
  recipes = {name: dict(seed=r[0], top=r[1], mask_shape=r[2], digest=bst.scene_digest(scenes[name]))
             for name, r in SCENES.items()}
  torch.save(dict(scenes=recipes, cases=cases), os.path.join(HERE, "bt_stab.pt"), pickle_protocol=4)


if __name__ == "__main__":
  main()
