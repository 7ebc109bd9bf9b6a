"""The library's 2-D encoder training forward and backward (csrc/encoder.cu, feature_network._EncoderFn) against the
float64 reference of the same computation (tests/encoder_ref.py), run on the device.

Precision "bf16" is compared with the reference in mode "kernel", which rounds the operands of exactly the products
the library puts on the tensor cores; precision "fp32" with mode "exact".  Compared: coarse, fine and the gradient
of every executed parameter (feature_network._EXECUTED).

The cases (encoder_ref.CASES) are chosen so that every dispatch branch and edge runs; rows are N H2 W2 at half
resolution (the stem) and N H4 W4 at quarter resolution (layer1, out_conv):
  minimum     1 x 8 x 8      16 / 4        2-wide planes under reflect padding, all SIMT, tile loads past the image
  small_odd   3 x 17 x 33    459 / 135     the largest shape whose tiles reach past the image; odd sizes, stride 2
  mixed       2 x 72 x 96    3456 / 864    the stem on the tensor cores, quarter resolution in SIMT
  below_2048  1 x 90 x 354   7965 / 2047   one row under the threshold
  at_2048     2 x 128 x 128  8192 / 2048   at the threshold, no partial tile; gradient of fine only
  ragged      3 x 150 x 206  23175 / 5928  partial last 128-row tile at both resolutions (7 and 40 rows)
  flat        2 x 64 x 96    3072 / 768    a constant image and a constant image plus 1e-4 noise: InstanceNorm
                                           variance far below eps
  bench       8 x 288 x 512  294912 / 73728  bench.py's train_step call: gradient of coarse only (the backward
                                           gets a zero d fine), many slabs per dW tile

Bars (encoder_ref.BARS): per precision and tensor, 2x the worst relative L2 error and 2x the worst max-abs ratio
measured over all cases of this file on an H100 80GB HBM3 (700 W), rounded up to one digit, at least 1e-5 (fp32) /
1e-4 (bf16); the comment beside each bar records the measured worst and its case.  Where no ReLU flips, both
precisions agree with the reference to about 1e-6 (fp32) and 1e-4 (bf16); coarse and fine to 1e-6 (8e-6 at 1 x 8 x 8).
The bars of the gradients (1e-3 to 2e-2 relative L2, up to 5e-2 max-abs, the same in both precisions) are set by
ReLU flips: a unit whose pre-activation lies within the fp32 / float64 difference of 0 passes its whole gradient on
one side and none on the other, and one flipped unit moves a weight gradient summed over 2047 rows by about
1 / sqrt(2047) = 2e-2 of its norm.  below_2048 sets most bars, and there precision fp32 measures the same numbers as
bf16 (its quarter-resolution products are SIMT in both): the errors start at layer1.2.bn1's ReLU (layer1.2.conv2,
bn2 and out_conv agree to 1e-6; layer1.2.bn1.bias 2.1e-2 and layer1.2.conv1.weight 2.4e-2 max-abs; 4e-3 relative L2
above).  29 of that ReLU's pre-activations lie within RELU_NEAR of their rounding scale of 0 (the test prints the
count over all ReLUs); flipping them in the reference moves exactly the same tensors, by 2.9e-2 / 9e-2 and 1.5e-2 on
conv1.weight, and nothing below.  The bf16 rounding itself adds at most 4e-3 (conv1.weight, ragged and bench).

Case "flat" compares only coarse and fine (FLAT_BAR, 2.7e-3 measured in both precisions) and requires every
gradient to be finite.  Its gradients cannot be computed in floating point: every plane of the constant image is
constant after every convolution, so each InstanceNorm sees variance 0 and multiplies the gradient by
rstd gamma = gamma / sqrt(1e-5), about 316, while the exact weight gradient of a layer feeding such a plane is a sum
over the plane that cancels to 0.  The rounding residue of that cancellation, amplified once per InstanceNorm, is the
whole result: the library is 7e7 times the norm of conv1.weight's float64 gradient off in both precisions, the
float32 reference 8e7 times, and two float64 evaluations (this reference and autograd through the oracle) already
differ by 16 % of their largest element.  The forward of the noisy image keeps only the bits its 1e-4 noise leaves
above fp32 resolution, hence 2.7e-3 rather than 1e-6.
"""

import copy

import pytest
import torch

import encoder_ref as er

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _library(c, prec):
  from dynibar_b200 import feature_network as fn, render_ray as rr
  mod = copy.deepcopy(c["mod"]).to(DEV).requires_grad_(True)
  with rr.precision_scope(prec):
    co, fi = mod(c["x"].to(DEV))
    loss = 0.0
    if c["gc"] is not None:
      loss = loss + (co * c["gc"].to(DEV)).sum()
    if c["gf"] is not None:
      loss = loss + (fi * c["gf"].to(DEV)).sum()
    loss.backward()
  torch.cuda.synchronize()
  params = dict(mod.named_parameters())
  for k, p in params.items():  # parameters the reference builds but never runs get no gradient
    assert (p.grad is not None) == (k in fn._EXECUTED), k
  got = {"coarse": co.detach(), "fine": fi.detach()}
  got.update({k: params[k].grad for k in fn._EXECUTED})
  return got


def _check(case, prec, got, ref):
  if case == "flat":
    for k, v in got.items():
      assert torch.isfinite(v).all(), k
    got, ref = ({k: d[k] for k in ("coarse", "fine")} for d in (got, ref))
  errs = er.errors(got, ref)
  r = er.ratios(prec, got, ref, flat=case == "flat")
  print("\nencoder %s %s: worst %s, %.2f of its bar" % (case, prec, *max(r.items(), key=lambda kv: kv[1])))
  for name, (rel, mx) in sorted(errs.items()):
    print("  ERR %s %s %s %.3e %.3e %.2f" % (case, prec, name, rel, mx, r[name]))
  bad = {k: errs[k] for k, v in r.items() if not v <= 1.0}
  assert not bad, (case, prec, bad)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("case", list(er.CASES))
def test_encoder_training_matches_reference(case, prec):
  c = er.make_case(case)
  got = _library(c, prec)
  stats = {}
  ref = er.reference(c, DEV, "kernel" if prec == "bf16" else "exact", stats=stats)
  print("\nencoder %s %s: %d of %d ReLU pre-activations within %.1e of their scale of 0" %
        (case, prec, sum(v[0] for v in stats.values()), sum(v[1] for v in stats.values()), er.RELU_NEAR))
  _check(case, prec, got, ref)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_three_calls_in_one_graph_sum_their_gradients(prec):
  """bench.py's train_step runs the encoder on three image sets and backpropagates through all three at once: the
  backward calls share one scratch buffer (workspace slot 3, grown for the largest call) and each reads its own saved
  activations.  The gradients must be the sum of three separate backward passes.  Image sets of 2, 3 and 1 images
  put the quarter-resolution products of the first two on the tensor cores (3072 and 4608 rows) and the third's in
  SIMT (1536 rows).  fp32: the float atomics' order is all that differs (1.1e-6 measured).  bf16: that order also
  moves operands across bf16 rounding boundaries, so two runs of the same separate passes differ by about as much as
  the library differs from the reference; the bar is the reference comparison's.  The test prints that run-to-run
  difference beside the one it checks."""
  from dynibar_b200 import feature_network as fn, render_ray as rr
  mod = er.make_model(7).to(DEV).requires_grad_(True)
  g = torch.Generator().manual_seed(8)
  imgs = [torch.rand(n, 3, 128, 192, generator=g).to(DEV) for n in (2, 3, 1)]
  gcs = [torch.randn(n, 32, 32, 48, generator=g).to(DEV) for n in (2, 3, 1)]
  params = dict(mod.named_parameters())

  def separate():
    mod.zero_grad(set_to_none=True)
    for im, gc in zip(imgs, gcs):  # .grad accumulates over the three passes
      (mod(im)[0] * gc).sum().backward()
    return {k: params[k].grad.clone() for k in fn._EXECUTED}

  with rr.precision_scope(prec):
    mod.zero_grad(set_to_none=True)
    sum((mod(im)[0] * gc).sum() for im, gc in zip(imgs, gcs)).backward()
    joint = {k: params[k].grad.clone() for k in fn._EXECUTED}
    sep, sep2 = separate(), separate()
  torch.cuda.synchronize()
  rel = lambda a, b: {k: ((a[k] - b[k]).norm() / b[k].norm()).item() for k in fn._EXECUTED}
  d, d2 = rel(joint, sep), rel(sep2, sep)
  print("\nthree calls in one graph, %s: worst relative L2 difference to three separate passes %.2e (%s); two runs "
        "of the separate passes: %.2e" % (prec, max(d.values()), max(d, key=d.get), max(d2.values())))
  bad = {k: v for k, v in d.items() if not v <= (1e-5 if prec == "fp32" else er.bar("bf16", k)[0])}
  assert not bad, bad
