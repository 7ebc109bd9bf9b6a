"""Host logic of monocular bullet-time sweeps (no GPU): the wander path and each camera's source views against the
reference's selection (tests/golden/bullet_time.pt, make_golden_bt.py), grouping a sweep into batched calls, the
pooled multi-camera batch builder, and the argument checks of the pooled C-ABI entry points, which run before any
CUDA call."""

import os

import numpy as np
import pytest
import torch

import scenes
from dynibar_b200 import bullet_time as bt
from dynibar_b200 import sample_ray as sr
from dynibar_b200 import synthetic

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bullet_time.pt")
H, W = 6, 8


@pytest.fixture(scope="module")
def golden():
  return torch.load(GOLDEN, weights_only=False)


def test_wander_path_matches_reference(golden):
  for case in golden["cases"]:
    got = np.array(bt.wander_path(case["llff_c2w"].numpy())).astype(np.float32)
    assert got.shape == (50, 3, 5)
    np.testing.assert_array_equal(got, case["wander"].numpy())


def test_select_source_views_matches_reference(golden):
  train, vv = golden["train_c2w"].numpy(), golden["src_vv_c2w"].numpy()
  fallbacks = 0
  for case in golden["cases"]:
    fallbacks += case["fallback"]
    for pose, want in zip(case["render_c2w"].numpy(), case["selections"]):
      got = bt.select_source_views(pose, train, vv, case["render_idx"], case["num_source_views"], case["max_range"],
                                   golden["num_vv"])
      assert got == tuple(list(w) for w in want), (case["render_idx"], got, want)
  assert fallbacks >= 1  # a case near the video's end, where the [::5] fallback fills the static views


def test_group_cameras_respects_both_limits(golden):
  train, vv = golden["train_c2w"].numpy(), golden["src_vv_c2w"].numpy()
  case = golden["cases"][1]
  sel = [bt.select_source_views(p, train, vv, case["render_idx"], 7, 10, golden["num_vv"])
         for p in case["render_c2w"].numpy()]
  groups = bt.group_cameras(sel)
  assert groups[0][0] == 0 and groups[-1][1] == len(sel)
  assert all(a[1] == b[0] for a, b in zip(groups, groups[1:]))
  for lo, hi in groups:
    assert 1 <= hi - lo <= 16
    assert len({("t", i) for t, _, _ in sel[lo:hi] for i in t} | {("vv", j) for _, v, _ in sel[lo:hi] for j in v}) <= 32
    assert len({i for _, _, s in sel[lo:hi] for i in s}) <= 32
  # a tight pool splits the sweep further
  tight = bt.group_cameras(sel, max_pool=15)
  assert len(tight) >= len(groups)
  with pytest.raises(ValueError, match="alone"):
    bt.group_cameras(sel, max_pool=4)


def _views(n, seed):
  g = torch.Generator().manual_seed(seed)
  batch, _, _, _, _, _ = synthetic.make_scene(H=H, W=W, V_dy=n, V_st=n, seed=seed)
  return batch["src_rgbs"][0] + 0.01 * torch.rand(batch["src_rgbs"][0].shape, generator=g), batch["src_cameras"][0]


def _pooled_case(dy_ids, st_ids, seed=5):
  """One get_all() batch per camera whose source views are drawn from per-identity views."""
  dy_keys = sorted({i for ids in dy_ids for i in ids}, key=repr)
  st_keys = sorted({i for ids in st_ids for i in ids}, key=repr)
  dy_r, dy_c = _views(len(dy_keys), seed)
  st_r, st_c = _views(len(st_keys), seed + 1)
  dy = {k: (dy_r[i], dy_c[i]) for i, k in enumerate(dy_keys)}
  st = {k: (st_r[i], st_c[i]) for i, k in enumerate(st_keys)}
  batch, _, _, _, _, _ = synthetic.make_scene(H=H, W=W, V_dy=2, V_st=2, seed=seed)
  data = scenes.sampler_data(batch, H, W, seed)
  K_mat = sr.parse_camera(batch["camera"])[2][0]
  out = []
  for k, (di, si) in enumerate(zip(dy_ids, st_ids)):
    c2w = torch.eye(4)
    c2w[0, 3] = 0.03 * k
    smp = sr.RaySamplerSingleImage(dict(data, camera=synthetic.camera_vector(H, W, K_mat, c2w)[None]), "cpu")
    b = smp.get_all()
    b["src_rgbs"] = torch.stack([dy[i][0] for i in di])[None]
    b["src_cameras"] = torch.stack([dy[i][1] for i in di])[None]
    b["static_src_rgbs"] = torch.stack([st[i][0] for i in si])[None]
    b["static_src_cameras"] = torch.stack([st[i][1] for i in si])[None]
    out.append(b)
  return out


TEMPORAL = [10, 11, 12, 13, 14, 15, 16]
DY_IDS = [TEMPORAL + [("vv", 2), ("vv", 5), ("vv", 1)], TEMPORAL + [("vv", 5), ("vv", 2), ("vv", 7)],
          TEMPORAL + [("vv", 0), ("vv", 2), ("vv", 5)]]
ST_IDS = [[3, 5, 7, 9, 11], [5, 7, 9, 11, 13], [3, 7, 11, 13, 17]]


def test_pooled_batch_round_trips():
  parts = _pooled_case(DY_IDS, ST_IDS)
  batch, counts, hw = sr.stack_pooled_ray_batches(parts, DY_IDS, ST_IDS)
  assert counts == [H * W] * 3 and hw == (H, W)
  assert batch["camera"].shape == (3, 34)
  assert batch["camera_index"].tolist() == [k for k in range(3) for _ in range(H * W)]
  # pools: deduplicated by identity, the temporal views first in slot order
  assert batch["src_cameras"].shape[1] == 7 + 5  # vv 0, 1, 2, 5, 7
  assert batch["static_src_cameras"].shape[1] == 7  # 3 5 7 9 11 13 17
  tv, ts = batch["src_views"], batch["static_src_views"]
  assert tv.dtype == torch.int32 and tv.shape == (3, 10) and ts.shape == (3, 5)
  assert all(tv[k, :7].tolist() == list(range(7)) for k in range(3))
  assert batch["src_view_ids"] == TEMPORAL + [("vv", 2), ("vv", 5), ("vv", 1), ("vv", 7), ("vv", 0)]
  assert batch["static_src_view_ids"] == [3, 5, 7, 9, 11, 13, 17]
  for k, p in enumerate(parts):
    for key, tkey in (("src", tv), ("static_src", ts)):
      sl = tkey[k].long()
      assert torch.equal(batch[key + "_rgbs"][:, sl], p[key + "_rgbs"]), (k, key)
      assert torch.equal(batch[key + "_cameras"][:, sl], p[key + "_cameras"]), (k, key)
  for k in ("ray_o", "ray_d", "uv_grid", "rgb"):
    for p, piece in zip(parts, batch[k].split(counts, 0)):
      assert torch.equal(piece, p[k]), k
  # equal identities with equal content in different tensors deduplicate too
  parts[1] = dict(parts[1], src_rgbs=parts[1]["src_rgbs"].clone())
  again, _, _ = sr.stack_pooled_ray_batches(parts, DY_IDS, ST_IDS)
  assert torch.equal(again["src_views"], tv)
  # one camera: its own views, the identity table
  one, _, _ = sr.stack_pooled_ray_batches(parts[:1], DY_IDS[:1], ST_IDS[:1])
  assert one["src_views"].tolist() == [list(range(10))] and one["static_src_views"].tolist() == [list(range(5))]


def test_pooled_batch_refusals():
  parts = _pooled_case(DY_IDS, ST_IDS)
  with pytest.raises(ValueError, match="1..16"):
    sr.stack_pooled_ray_batches(parts[:1] * 17, DY_IDS[:1] * 17, ST_IDS[:1] * 17)
  # temporal slots that differ between cameras
  bad = [DY_IDS[0], [9] + TEMPORAL[1:] + DY_IDS[1][7:], DY_IDS[2]]
  with pytest.raises(ValueError, match="temporal slots differ"):
    sr.stack_pooled_ray_batches(_pooled_case(bad, ST_IDS), bad, ST_IDS)
  # a depth range that differs
  other = dict(parts[2], depth_range=parts[2]["depth_range"] * 1.5)
  with pytest.raises(ValueError, match="depth_range"):
    sr.stack_pooled_ray_batches(parts[:2] + [other], DY_IDS, ST_IDS)
  # equal identity, different content
  moved = parts[1]["static_src_rgbs"].clone()
  moved[0, 0] += 0.25
  with pytest.raises(ValueError, match="equal identities"):
    sr.stack_pooled_ray_batches(parts[:1] + [dict(parts[1], static_src_rgbs=moved)] + parts[2:], DY_IDS, ST_IDS)
  # a pool of more than 32 views
  st_many = [list(range(0, 15)), list(range(15, 30)), list(range(30, 45))]
  with pytest.raises(ValueError, match="at most 32"):
    sr.stack_pooled_ray_batches(_pooled_case(DY_IDS, st_many), DY_IDS, st_many)


@pytest.mark.parametrize("K,pool,V,with_index,with_tbl,msg", [
    (17, 8, 5, True, True, b"K = 17"), (0, 8, 5, True, True, b"K = 0"),
    (3, 8, 5, False, True, b"per-ray camera index"), (3, 8, 5, True, False, b"view table"),
    (3, 33, 5, True, True, b"pool of 33"), (3, 0, 5, True, True, b"pool of 0"),
    (3, 8, 33, True, True, b"33 view slots"), (3, 8, 0, True, True, b"0 view slots")])
def test_pooled_entry_points_check_arguments_before_any_cuda_call(K, pool, V, with_index, with_tbl, msg):
  from dynibar_b200 import _lib
  lib = _lib.lib
  fake = 0x1000  # never dereferenced: the checks return first
  idx = fake if with_index else None
  tbl = fake if with_tbl else None
  R, S = 8, 16
  rc = lib.dyn_project_gather_tbl(fake, None, fake, K, idx, tbl, pool, fake, fake, fake, V, R, S, H, W, 32, H // 2,
                                  W // 2, fake, fake, fake, fake, None)
  assert rc == -1 and msg in lib.dyn_last_error()
  rc = lib.dyn_plucker_src_tbl(fake, fake, pool, K, idx, tbl, V, R, S, fake, None)
  assert rc == -1 and msg in lib.dyn_last_error()
  # the fused forms take at most 16 slots per camera
  Vf = 17 if V == 33 else V
  msg_f = b"17 view slots" if V == 33 else msg
  rc = lib.dyn_net_static_fused_tbl(None, fake, fake, fake, fake, K, idx, tbl, pool, fake, fake, fake, R, S, Vf, H, W,
                                    32, H // 2, W // 2, fake, fake, fake, 1 << 20, None)
  assert rc == -1 and msg_f in lib.dyn_last_error()
  rc = lib.dyn_net_dynamic_fused_tbl(None, fake, fake, fake, fake, K, idx, tbl, pool, fake, fake, fake, 0.5, R, S, Vf,
                                     H, W, 32, H // 2, W // 2, fake, fake, fake, 1 << 20, None)
  assert rc == -1 and msg_f in lib.dyn_last_error()
