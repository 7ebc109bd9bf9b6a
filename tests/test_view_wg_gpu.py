"""The warpgroup per-view kernel (csrc/view_wg.cu, the library default) against the twin-warp kernel
(csrc/view_twin.cu): same math with accumulators in registers, biases added in fp32 in the epilogues and
hidden activations handed on as bf16 register operands.  Differences come only from the fp32 summation order
and the bf16 re-rounding of activations it can flip (tolerances below)."""

import pytest
import torch

from dynibar_b200 import _lib, synthetic
from util import assert_close_frac

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _inputs(V_dy, V_st, rays, S, seed, stress=False, mask_rgb=0):
  from dynibar_b200 import render_ray as rr
  batch, feat_c, feat_f, frame, t, offs = synthetic.make_scene(H=72, W=96, V_dy=V_dy, V_st=V_st, rays=rays,
                                                               seed=seed, stress=stress)
  args = synthetic.make_args(1, mask_rgb)
  model, args = synthetic.make_model(S, 0, args=args, seed=seed, mono=True)
  d = lambda x: synthetic.to_device(x, DEV)
  b, fc = d(batch), d(feat_c)
  m = synthetic.model_to(model, DEV)
  pts, z, s = rr.sample_along_camera_ray(b["ray_o"], b["ray_d"], b["depth_range"], S, True, True)
  g = torch.Generator(device=DEV).manual_seed(seed)
  seq = pts[None] + 0.02 * torch.randn(V_dy, rays, S, 3, device=DEV, generator=g)
  return b, fc, m, pts, seq, float(t[0].float())


def _run(b, fc, m, pts, seq, tt, kernel):
  """Both fused aggregation nets with per-view kernel `kernel` (dyn_debug_set_view_kernel)."""
  from dynibar_b200 import render_ray as rr
  _lib.lib.dyn_debug_set_view_kernel(kernel)
  try:
    ray_dir = torch.nn.functional.normalize(b["ray_d"], dim=-1)
    raw_st, m_st = rr.net_static_fused(m.net_coarse_st, pts, b["ray_o"], b["ray_d"], b["camera"],
                                       b["static_src_rgbs"], b["static_src_cameras"],
                                       rr.featmaps_channels_last(fc[2]))
    raw_dy, m_dy = rr.net_dynamic_fused(m.net_coarse_dy, pts, seq, ray_dir, b["camera"], b["src_rgbs"],
                                        b["src_cameras"], rr.featmaps_channels_last(fc[0]), tt)
    torch.cuda.synchronize()
  finally:
    _lib.lib.dyn_debug_set_view_kernel(-1)  # back to the library default
  return raw_st, m_st, raw_dy, m_dy


@pytest.mark.parametrize("V_dy,V_st,rays,S,stress,mask_rgb", [
    (8, 8, 300, 64, False, 0),     # the benchmark's view counts, several 128-row iterations, ragged tail
    (7, 11, 130, 32, True, 1),     # eval_nvidia.py:92-119 view counts: 8 and 16 view slots, masks stressed
    (10, 15, 70, 64, False, 1),    # BASELINE config 4
    (3, 2, 33, 16, True, 0),       # tiny: a single partially filled tile
    (16, 16, 40, 32, False, 0),    # full 16-slot groups
])
def test_wg_kernel_matches_twin_kernel(V_dy, V_st, rays, S, stress, mask_rgb):
  inp = _inputs(V_dy, V_st, rays, S, seed=V_dy * 100 + V_st, stress=stress, mask_rgb=mask_rgb)
  w = _run(*inp, kernel=-1)
  t = _run(*inp, kernel=0)
  assert torch.equal(w[1], t[1]) and torch.equal(w[3], t[3])  # projector masks: pure fp32 geometry
  for name, a, b, mask in (("st", w[0], t[0], w[1]), ("dy", w[2], t[2], w[3])):
    assert torch.isfinite(a[..., :3]).all()
    valid = (mask.sum(2) > 0)[..., 0]
    assert (a[..., 3][~valid] == -1e9).all() and (b[..., 3][~valid] == -1e9).all()
    assert_close_frac("rgb_" + name, a[..., :3][valid], b[..., :3][valid], rtol=0, atol=4e-3, max_bad_frac=1e-3)
    assert_close_frac("sigma_" + name, a[..., 3][valid], b[..., 3][valid], rtol=0, atol=2e-2, max_bad_frac=1e-3)


def _assert_deterministic_and_chunk_invariant(kernel):
  b, fc, m, pts, seq, tt = _inputs(8, 8, 520, 32, seed=5)
  full = _run(b, fc, m, pts, seq, tt, kernel=kernel)
  again = _run(b, fc, m, pts, seq, tt, kernel=kernel)
  for x, y in zip(full, again):
    assert torch.equal(x, y)
  n = 200
  bs = dict(b)
  for k in ("ray_o", "ray_d", "uv_grid"):
    bs[k] = b[k][:n].contiguous()
  part = _run(bs, fc, m, pts[:n].contiguous(), seq[:, :n].contiguous(), tt, kernel=kernel)
  for x, y in zip(full, part):
    assert torch.equal(x[:n], y)


def test_wg_kernel_is_deterministic_and_chunk_invariant():
  """rows are independent: evaluating a prefix of the rays gives bit-identical results (different grid size,
  different pairing of half-tiles in a CTA), and repeated launches are bit-identical."""
  _assert_deterministic_and_chunk_invariant(-1)


def test_twin_kernel_is_deterministic_and_chunk_invariant():
  """the same for the twin-warp kernel the default is compared against (different grid size, different
  tiles)."""
  _assert_deterministic_and_chunk_invariant(0)


def test_removed_view_kernels_fail_loudly():
  """selectors 1 - 3 named kernels that have been removed: a fused render with one of them fails and says
  so instead of running another kernel under that name."""
  inp = _inputs(3, 2, 33, 16, seed=7)
  for kernel, what in ((1, "quad-schedule"), (2, "sub-round pipelined twin"), (3, "sub-round pipelined twin")):
    with pytest.raises(RuntimeError, match="per-view kernel %d \\(the %s kernel\\) has been removed" % (kernel, what)):
      _run(*inp, kernel=kernel)
