"""A ray's per-point outputs do not depend on where the fused per-point stage places it.

When S divides 128 the whole per-point stage (point1, the ray-transformer attention, point2) runs as one kernel in
which each 128-row iteration is split between two 64-row warpgroups.  Dropping the first ray of a batch moves every
other ray by S rows: at S = 16 to other keys of its warpgroup (and some rays to the other warpgroup), at S = 64 to
the other warpgroup, at S = 128 to another iteration.  The raw output (dynamic net) or GW and sigma (static net) of
each ray must stay bit-identical, which a camera rendered inside a batch relies on.  dyn_debug_point_chain runs the
product kernel when it is asked for none of the exchanged values (capture=False here) and its capturing
instantiation otherwise: both are checked."""

import pytest
import torch

import point_stage_ref as psr
from dynibar_b200 import _lib, weights
from test_point_stage_gpu import DEV, _nan, _net, run_chain

pytestmark = pytest.mark.gpu

def run_product(net, kind, G, nvalid, pts, ray_dir, R, S):
  """dyn_debug_point_chain without g2, Q, K, V, O: the product kernel -> out_a, out_b."""
  P = R * S
  packed = weights.packed_of(net, torch.device(DEV))
  d = lambda x: x.to(DEV).contiguous()
  Gd, nvd, ptd, rdd = d(G), d(nvalid), d(pts), d(ray_dir)
  out = {"out_a": _nan(P, 128 if kind == "static" else 4), "out_b": _nan(P)}
  pws = torch.zeros(S * 128, device=DEV)
  _lib.check(_lib.lib.dyn_debug_point_chain(
      packed.handle, Gd.data_ptr(), nvd.data_ptr(), ptd.data_ptr(), rdd.data_ptr(), R, S,
      None, None, None, None, None, out["out_a"].data_ptr(), out["out_b"].data_ptr(), pws.data_ptr(), _lib.stream()))
  torch.cuda.synchronize()
  return out


@pytest.mark.parametrize("capture", [False, True])
@pytest.mark.parametrize("kind", ["dynamic", "static"])
@pytest.mark.parametrize("S,R", [(16, 37), (64, 37), (128, 9)])
def test_ray_outputs_do_not_depend_on_position(kind, S, R, capture):
  net = _net(kind)
  run = run_chain if capture else run_product
  G, nvalid, pts, ray_dir = psr.make_point_inputs(R + 1, S, seed=11 * S + R)
  full = run(net, kind, G, nvalid, pts, ray_dir, R + 1, S)
  shifted = run(net, kind, G[S:], nvalid[S:], pts[S:], ray_dir[1:], R, S)
  keys = ("out_a",) if kind == "dynamic" else ("out_a", "out_b")
  for k in keys:
    a, b = full[k][S:], shifted[k]
    assert torch.isfinite(a).all(), k
    assert torch.equal(a, b), (k, (a - b).abs().max().item())


@pytest.mark.parametrize("kind", ["dynamic", "static"])
@pytest.mark.parametrize("S,R", [(16, 37), (64, 37), (128, 9)])
def test_product_kernel_matches_capturing_kernel(kind, S, R):
  """The product kernel (no stores of g2, Q, K, V, O) and its capturing twin: same outputs, bit for bit."""
  net = _net(kind)
  G, nvalid, pts, ray_dir = psr.make_point_inputs(R, S, seed=7 * S + R)
  a = run_product(net, kind, G, nvalid, pts, ray_dir, R, S)
  b = run_chain(net, kind, G, nvalid, pts, ray_dir, R, S)
  for k in (("out_a",) if kind == "dynamic" else ("out_a", "out_b")):
    assert torch.equal(a[k], b[k]), (k, (a[k] - b[k]).abs().max().item())
