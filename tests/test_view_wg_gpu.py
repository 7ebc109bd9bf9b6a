"""The warpgroup per-view kernel (csrc/view_wg.cu, the library default) against the twin-warp kernel
(csrc/view_twin.cu): same math with accumulators in registers, biases added in fp32 in the epilogues and
hidden activations handed on as bf16 register operands.  Differences come only from the fp32 summation order
and the bf16 re-rounding of activations it can flip (tolerances of test_view_quad_gpu.py)."""

import pytest
import torch

from test_view_quad_gpu import _inputs, _run
from util import assert_close_frac

pytestmark = pytest.mark.gpu


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


def test_wg_kernel_is_deterministic_and_chunk_invariant():
  """rows are independent: evaluating a prefix of the rays gives bit-identical results (different grid size,
  different pairing of half-tiles in a CTA), and repeated launches are bit-identical."""
  b, fc, m, pts, seq, tt = _inputs(8, 8, 520, 32, seed=5)
  full = _run(b, fc, m, pts, seq, tt, kernel=-1)
  again = _run(b, fc, m, pts, seq, tt, kernel=-1)
  for x, y in zip(full, again):
    assert torch.equal(x, y)
  n = 200
  bs = dict(b)
  for k in ("ray_o", "ray_d", "uv_grid"):
    bs[k] = b[k][:n].contiguous()
  part = _run(bs, fc, m, pts[:n].contiguous(), seq[:, :n].contiguous(), tt, kernel=-1)
  for x, y in zip(full, part):
    assert torch.equal(x[:n], y)
