"""The fused per-view stage (csrc/view_wg.cu, and the twin-warp kernel csrc/view_twin.cu) against a float64
reference that rounds to bf16 where the kernel does (tests/view_stage_ref.py, mode="kernel").

dyn_debug_set_view_capture copies what the stage hands to the per-point stage and the blending head (G, nvalid,
X, vis2, mask_eff, ray_diff, rgb_in) out of every internal chunk of a fused render.  The cases cover 8- and
16-slot kernels with full and padded slot groups, launches that end in a partial half-tile, the benchmark shape
(several iterations per persistent CTA), a launch of two internal chunks, points behind or far from a source
camera, with zero, one and all valid views, taps across the feature-map edge, exact-black source pixels under
mask_rgb, anti-aliased pooling on, off and with |s| = 0, virtual views of the dynamic net, positional-encoding
arguments up to 16 x 30 rad, and weights large enough to drive the ELUs and sigmoids out of their linear range.
"""

import pytest
import torch

import view_stage_ref as vr
from dynibar_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

CASES = {
    # view counts: 8-slot (1, 2, 7, 8) and 16-slot (9, 11, 16) kernels; P * VP a multiple of neither 64 nor 128
    "V1": dict(V=1, rays=13, S=5, seed=21),
    "V2": dict(V=2, rays=13, S=5, seed=22),
    "V7": dict(V=7, rays=17, S=9, seed=23),
    "V8": dict(V=8, rays=17, S=9, seed=24),
    "V9": dict(V=9, rays=11, S=7, seed=25),
    "V11": dict(V=11, rays=11, S=7, seed=26),
    "V16": dict(V=16, rays=9, S=7, seed=27),
    # P = 5 < 8: one partial half-tile
    "tiny": dict(V=3, rays=1, S=5, seed=28),
    # the benchmark shape: ~1200 iterations of 128 rows, several per persistent CTA
    "bench": dict(V=8, rays=300, S=64, seed=29),
    # two internal chunks (net_rows_per_chunk(128, 16) = 2048 rays)
    "two_chunks": dict(V=16, rays=2050, S=128, seed=30, H=48, W=64),
    # a camera behind the near samples, far-off cameras, H and W not divisible by 4
    "stress": dict(V=8, rays=160, S=32, seed=31, stress=True, H=70, W=94),
    # exact-black source regions: mask_rgb rejects views the projector accepts
    "mask_rgb": dict(V=8, rays=96, S=16, seed=32, mask_rgb=1, black=True, stress=True),
    "no_aa": dict(V=9, rays=40, S=16, seed=33, anti_alias=0, mask_rgb=1, black=True),
    "s_zero": dict(V=8, rays=40, S=16, seed=34, s_zero=True),
    # dynamic virtual views (no displacement), far plane 30
    "vv_far": dict(V=10, rays=60, S=32, seed=35, num_vv=3, far=30.0),
    # per-view layer weights x3: activations leave the near-linear range
    "hot": dict(V=8, rays=60, S=16, seed=36, weight_scale=3.0, stress=True),
}
N_RANDOM = 256  # sampled points per case (plus edge points, see _sample)
RC_RAYS = 2048  # rays per internal chunk at S = 128, V = 16


def _capture(kind, net, sc, kernel):
  """One fused render of net `kind` with per-view kernel `kernel`; returns the projector mask and the
  captured per-view outputs (CUDA tensors)."""
  from dynibar_b200 import render_ray as rr
  d = lambda t: t.to(DEV)
  V = sc["src_cams"].shape[0]
  P = sc["pts"].shape[0]
  S = sc["S"]
  R = P // S
  nan = lambda *shape: torch.full(shape, float("nan"), device=DEV)
  cap = {"G": nan(P, vr.GCOLS), "nvalid": nan(P), "X": nan(P, V, 128), "vis2": nan(P, V),
         "mask_eff": nan(P, V), "ray_diff": nan(P, V, 4), "rgb_in": nan(P, V, 3)}
  order = ("G", "nvalid", "X", "vis2", "mask_eff", "ray_diff", "rgb_in")
  net = net.to(DEV)
  pts = d(sc["pts"]).reshape(R, S, 3)
  cams, rgbs = d(sc["src_cams"])[None], d(sc["src_rgbs"])[None]
  feat = rr.featmaps_channels_last(d(sc["featmaps"]))
  _lib.lib.dyn_debug_set_view_kernel(kernel)
  _lib.lib.dyn_debug_set_view_capture(*[cap[k].data_ptr() for k in order])
  try:
    if kind == "static":
      _, mask = rr.net_static_fused(net, pts, d(sc["ray_o"]), d(sc["ray_d"]), d(sc["query_cam"])[None], rgbs, cams,
                                    feat)
    else:
      ray_dir = torch.nn.functional.normalize(d(sc["ray_d"]), dim=-1)
      seq = d(sc["pts_seq"]).reshape(V, R, S, 3)
      _, mask = rr.net_dynamic_fused(net, pts, seq, ray_dir, d(sc["query_cam"])[None], rgbs, cams, feat,
                                     sc["time"])
    torch.cuda.synchronize()
  finally:
    _lib.lib.dyn_debug_set_view_capture(None, None, None, None, None, None, None)
    _lib.lib.dyn_debug_set_view_kernel(-1)
  return mask.reshape(P, V), cap


def _sample(P, S, mask_proj, seed):
  """Random points, the first and last point, both sides of every internal chunk boundary, and points with
  zero, one and all valid views."""
  g = torch.Generator().manual_seed(seed)
  idx = [torch.randperm(P, generator=g)[:N_RANDOM], torch.tensor([0, P - 1])]
  for b in range(RC_RAYS * S, P, RC_RAYS * S):
    idx.append(torch.arange(b - 2 * S, min(P, b + 2 * S)))
  nv = mask_proj.sum(1)
  V = mask_proj.shape[1]
  for want in (0, 1, V):
    hit = torch.nonzero(nv == want)[:, 0]
    idx.append(hit[torch.randperm(hit.numel(), generator=g)[:16]])
  return torch.unique(torch.cat(idx))


def compare(case, kind, kernel):
  """Runs one case -> per output (max |err|, max err / tolerance), facts about the sampled points, and the
  captured and reference values of the compared points."""
  nets, st, dy = vr.make_case(**CASES[case])
  sc = st if kind == "static" else dy
  mask_proj, cap = _capture(kind, nets[kind], sc, kernel)
  P, V = mask_proj.shape
  mask_proj = mask_proj.cpu()
  G = cap["G"]
  facts = {"G_pad": bool((G[:, 257:264] == 0).all() and (G[:, 264:266] == 1).all() and (G[:, 266:] == 0).all()),
           "all_rows_written": bool(torch.isfinite(G).all() and torch.isfinite(cap["nvalid"]).all())}
  if kind == "static":
    facts["all_rows_written"] &= all(bool(torch.isfinite(cap[k]).all()) for k in ("X", "vis2", "mask_eff"))
  else:  # the dynamic net writes only G, nvalid and the projector mask
    facts["untouched"] = all(bool(torch.isnan(cap[k]).all()) for k in ("X", "vis2", "mask_eff", "ray_diff", "rgb_in"))
  idx = _sample(P, sc["S"], mask_proj, CASES[case]["seed"])
  ref = vr.view_stage(kind, nets[kind].cpu().state_dict(), sc, idx=idx, mode="kernel")
  got = {k: v[idx.to(DEV)].cpu().double() for k, v in cap.items()}
  amb = ref["ambiguous"]
  masks = [(mask_proj[idx].double(), ref["mask_proj"])]
  if kind == "static":
    masks.append((got["mask_eff"], ref["mask_eff"]))
  facts["mask_mismatch_outside_ambiguous"] = sum(int(((a != b) & ~amb).sum()) for a, b in masks)
  keep = ~amb.any(1)
  facts["n_points"] = int(idx.numel())
  facts["n_ambiguous"] = int((~keep).sum())
  nv = ref["nvalid"][keep]
  facts["nvalid_classes"] = sorted({0 if x == 0 else (1 if x == 1 else (V if x == V else -1)) for x in nv.tolist()})
  facts["mask_eff_differs"] = bool((ref["mask_eff"] != ref["mask_proj"]).any())
  column = ("wg" if kernel < 0 else "twin") + ("_hot" if CASES[case].get("weight_scale", 1.0) != 1.0 else "")
  errs = vr.errors(got, ref, kind, keep, column)
  return errs, facts, (got, ref, keep)


@pytest.mark.parametrize("kernel", [-1, 0], ids=["wg", "twin"])
@pytest.mark.parametrize("kind", ["static", "dynamic"])
@pytest.mark.parametrize("case", list(CASES))
def test_view_stage_matches_reference(case, kind, kernel):
  errs, facts, _ = compare(case, kind, kernel)
  assert facts["all_rows_written"] and facts["G_pad"], facts
  if kind == "dynamic":
    assert facts["untouched"], facts
  assert facts["mask_mismatch_outside_ambiguous"] == 0, facts
  assert facts["n_ambiguous"] <= max(2, facts["n_points"] // 50), facts
  # compared points with zero, one and all valid views (the static rig of "stress" has none with one)
  V = CASES[case]["V"]
  if (case, kind) in (("stress", "dynamic"), ("mask_rgb", "static"), ("bench", "static"), ("bench", "dynamic")):
    assert {0, 1, V} <= set(facts["nvalid_classes"]), facts
  if (case, kind) == ("stress", "static"):
    assert {0, V} <= set(facts["nvalid_classes"]), facts
  if case in ("mask_rgb", "no_aa") and kind == "static":
    assert facts["mask_eff_differs"], facts
  bad = {k: v for k, v in errs.items() if v[1] > 1.0}
  assert not bad, "outputs out of tolerance (max |err|, err / tol): %s" % bad
