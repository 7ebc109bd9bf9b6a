"""The fused per-point stage (point_fused_wg_kernel) at point counts where every persistent CTA runs about 20
iterations, so each CTA's weight ring and G tile wrap many times, at both key widths (KEYS = 128 at S = 128, 64
otherwise) and for both nets.

dyn_debug_point_chain runs the product kernel when no captures are asked for.  Its result must not depend on the
launch: two launches on the same inputs are bit-identical, and so is the same run cut into pieces of fewer
iterations than there are SMs, where every CTA runs at most one iteration from the ring's first slot and every
piece ends in its own ragged tail.  test_point_stage_gpu.py checks such short runs against the float64 reference.
"""

import pytest
import torch

import point_stage_ref as psr
from test_ray_stage_gpu import run_product
from test_point_stage_gpu import _net

pytestmark = pytest.mark.gpu

# (S, R, piece): the whole run is about 2640 iterations of 128 rows (20 per CTA on 132 SMs) and not a whole number
# of rounds; a piece is 101 (S = 128), 100.5 (S = 64) or 125.1 (S = 16) iterations.  S = 128 runs KEYS = 128,
# S = 64 and 16 KEYS = 64 (the last with 8 rays per warpgroup and a last iteration of 48 rows).
CASES = [(128, 2641, 101), (64, 5281, 201), (16, 20011, 1001)]


@pytest.mark.parametrize("kind", ["dynamic", "static"])
@pytest.mark.parametrize("S,R,piece", CASES)
def test_fused_stage_is_launch_invariant(kind, S, R, piece):
  net = _net(kind)
  G, nvalid, pts, ray_dir = psr.make_point_inputs(R, S, seed=3 * S + R)
  keys = ("out_a",) if kind == "dynamic" else ("out_a", "out_b")
  full = run_product(net, kind, G, nvalid, pts, ray_dir, R, S)
  for k in keys:
    assert torch.isfinite(full[k]).all(), k
  again = run_product(net, kind, G, nvalid, pts, ray_dir, R, S)
  for k in keys:
    assert torch.equal(again[k], full[k]), "%s: two launches on the same inputs differ" % k
  for lo in range(0, R, piece):
    hi = min(R, lo + piece)
    part = run_product(net, kind, G[lo * S:hi * S], nvalid[lo * S:hi * S], pts[lo * S:hi * S], ray_dir[lo:hi],
                       hi - lo, S)
    for k in keys:
      diff = part[k] != full[k][lo * S:hi * S]
      diff = diff.reshape(diff.shape[0], -1).any(1)
      assert not diff.any(), "%s: rays %d .. %d run alone: %d points differ from the whole run (first %d)" % (
          k, lo, hi - 1, int(diff.sum()), lo * S + int(torch.nonzero(diff)[0, 0]))
