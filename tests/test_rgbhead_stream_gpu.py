"""The streaming static blending head (rgbhead_wg_kernel) at point counts where every persistent CTA runs many
iterations, so the X / GW ring of each CTA wraps several times and the per-row inputs of each iteration are
loaded during the one before it.

dyn_debug_rgb_head runs the product's kernel.  Its result must not depend on the launch: two launches on the same
inputs are bit-identical, and so is the same run cut into pieces of fewer iterations than there are SMs, where
every CTA runs one iteration from the ring's first slot, the points sit at other rows of their tiles, and every
piece ends in its own ragged tail.  test_point_stage_gpu.py checks that regime against the float64 reference.
"""

import pytest
import torch

import point_stage_ref as psr
from dynibar_b200 import _lib, synthetic, weights

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def run_rgb_head(net, inp, lo, hi, V):
  """raw [hi - lo, 4] of points lo .. hi - 1 run on their own."""
  packed = weights.packed_of(net, torch.device(DEV))
  d = {k: v[lo:hi].contiguous() for k, v in inp.items()}
  raw = torch.full((hi - lo, 4), float("nan"), device=DEV)
  _lib.check(_lib.lib.dyn_debug_rgb_head(packed.handle, *[d[k].data_ptr() for k in (
      "X", "vis2", "ray_diff", "mask_eff", "rgb_in", "GW", "sigma")], hi - lo, V, raw.data_ptr(), _lib.stream()))
  torch.cuda.synchronize()
  return raw


# (V, P, piece): V = 8 runs 8 view slots per point, V = 11 runs 16.  P * VP / 128 is about 2500 iterations (about
# 19 per CTA on 132 SMs) and not a whole number; a piece is 63 or 88 iterations, the last one partly filled.
CASES = [(8, 40003, 1001), (11, 20011, 701)]


@pytest.mark.parametrize("V,P,piece", CASES)
def test_streaming_head_is_launch_invariant(V, P, piece):
  model, _ = synthetic.make_model(64, 0, mono=True, seed=4)
  net = model.net_coarse_st.to(DEV)
  inp = {k: v.to(DEV) for k, v in psr.make_head_inputs(P, V, seed=7 * V + 1).items()}
  full = run_rgb_head(net, inp, 0, P, V)
  assert torch.isfinite(full).all()
  assert torch.equal(full[:, 3], inp["sigma"]), "sigma is not passed through"
  assert torch.equal(run_rgb_head(net, inp, 0, P, V), full), "two launches on the same inputs differ"
  for lo in range(0, P, piece):
    hi = min(P, lo + piece)
    diff = (run_rgb_head(net, inp, lo, hi, V) != full[lo:hi]).any(1)
    assert not diff.any(), "points %d .. %d run alone: %d differ from the whole run (first %d)" % (
        lo, hi - 1, int(diff.sum()), lo + int(torch.nonzero(diff)[0, 0]))
