"""The library's training backward of DynibarDynamic, DynibarStatic and the MotionMLP against the float64 reference
of the same computation (tests/train_stage_ref.py), run on the device.

Precision "bf16" is compared with the reference in mode "kernel", which rounds the operands of exactly the
products the library puts on the tensor cores; precision "fp32" with mode "exact".  Every output and every
gradient the library returns is compared: raw / coeff, each parameter (with `s` of the anti-aliased pooling), d
rgb_feat, d pts, d xyzt.

The cases are chosen so that every dispatch branch (train_stage_ref.dispatch) runs:
  all_simt     P < 128: precision bf16 entirely in SIMT
  fwd_tc_only  forward on the tensor cores, M = 1920 < 2048: backward in SIMT
  view_tc      per-view products on the tensor cores, per-point ones in SIMT
  ragged       P = 2096, M = 23 056 (not multiples of 64), every per-point and per-view product on the tensor cores
  per_ray_tc   R >= 2048: the per-ray products (dynamic rgb_fc.0's direction columns, static ref_feature_fc)
  v1, v16      the group sums over 1 and 16 views
  bench_like   several slabs per dW tile (float atomics from many CTAs), anti-aliasing and mask_rgb on
  MotionMLP    N across the forward (128) and backward (2048) thresholds, coeff_linear's dIn at 12 (SIMT) and 18
               (tensor cores) columns, the 388-column split of pts_linears.5

Bars (train_stage_ref.BARS): per net, precision and tensor, 2x the worst relative L2 error and 2x the worst
max-abs ratio measured over all cases of this file on an H100 80GB HBM3 (700 W), rounded up to one digit, at least
1e-5 (fp32) / 1e-4 (bf16); the comment beside each bar records the measured worst and its case.  fp32 agrees to
about 1e-6 except the column sums that cancel (vis_fc2.2.bias 2e-4, vis_fc2.0.bias, the blending head's biases).
bf16 does not reach the 1e-3 hoped for: the measured worst is 2e-3 to 6e-3 for the per-view and trunk layers
(1e-2 to 5e-2 for the blending head and for vis_fc2.2's bias, a sum over views that cancels).  This is double
rounding that compounds: where the GPU's fp32 value and the reference's float64 value of an operand straddle a
bf16 rounding boundary they round to neighbouring bf16 values, and each product's difference raises the chance of
such a split in the next one, so after a few layers the difference is a fair fraction of one bf16 ulp.  Running
the same reference in float32 on the CPU (reference(..., dtype=torch.float32)) gives the same 4e-3 against float64
on the ragged case, so the size is the arithmetic's, not a wiring error's.  The MotionMLP's bars are set by ReLU
flips, a unit whose pre-activation lies within the fp32 / float64 difference of 0 passing its whole gradient on one
side and none on the other.  In fp32 (bars up to 1e-2) that difference is fp32 arithmetic's: the same reference in
float32 on the CPU reproduces pts_linears.0.weight's 4.5e-3 at N = 2049.  In bf16 (bars 2e-2) the operands' double
rounding widens it; about 9e-5 of the pre-activations lie within 2^-16 of their scale of 0 (the test prints the
count), and sqrt(9e-5) = 9e-3 in L2.
"""

import copy

import pytest
import torch

import train_stage_ref as tsr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _library(c, prec):
  from dynibar_b200 import autograd as ag
  mod = copy.deepcopy(c["mod"]).to(DEV).requires_grad_(True)
  d = lambda x: x.to(DEV)
  if c["kind"] == "motion":
    x = d(c["xyzt"]).requires_grad_(True)
    out = ag.motion_mlp(mod, x, precision=prec)
    ins = {"xyzt": x}
  elif c["kind"] == "dynamic":
    pts, feat = d(c["pts"]).requires_grad_(True), d(c["feat"]).requires_grad_(True)
    out = ag.net_dynamic(mod, pts, feat, d(c["ray_dir"]), d(c["mask"]), torch.tensor([c["t"]]), precision=prec)
    ins = {"pts": pts, "rgb_feat": feat}
  else:
    feat = d(c["feat"]).requires_grad_(True)
    out = ag.net_static(mod, d(c["pts"]), d(c["ref_rays"]), d(c["src_rays"]), feat, d(c["ray_diff"]), d(c["mask"]),
                        precision=prec)
    ins = {"rgb_feat": feat}
  (out * d(c["gen"])).sum().backward()
  got = {"out": out.detach()}
  got.update({k: p.grad for k, p in mod.named_parameters()})
  got.update({k: v.grad for k, v in ins.items()})
  return got


def _check(kind, case, prec, got, ref, V=None):
  errs = tsr.errors(kind, got, ref, V)
  r = tsr.ratios(kind, prec, got, ref, V)
  print("\n%s %s %s: worst %s, %.2f of its bar" % (kind, case, prec, *max(r.items(), key=lambda kv: kv[1])))
  for name, (rel, mx) in sorted(errs.items()):
    print("  ERR %s %s %s %s %.3e %.3e" % (kind, case, prec, name, rel, mx))
  bad = {k: (errs[k], tsr.bar(kind, prec, k)) for k, v in r.items() if not v <= 1.0}
  assert not bad, (kind, case, prec, bad)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("case", list(tsr.NET_CASES))
@pytest.mark.parametrize("kind", ["dynamic", "static"])
def test_net_training_matches_reference(kind, case, prec):
  R, S, V, aa, mrgb = tsr.NET_CASES[case]
  c = tsr.make_net_case(kind, R, S, V, aa, mrgb, seed=R + V)
  got = _library(c, prec)
  ref = tsr.reference(c, DEV, "kernel" if prec == "bf16" else "exact")
  _check(kind, case, prec, got, ref, V)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("case", list(tsr.MOTION_CASES))
def test_motion_training_matches_reference(case, prec):
  N, nb = tsr.MOTION_CASES[case]
  c = tsr.make_motion_case(N, nb, seed=N + nb)
  got = _library(c, prec)
  stats = {}
  ref = tsr.reference(c, DEV, "kernel" if prec == "bf16" else "exact", stats=stats)
  near = sum(v[0] for v in stats.values())
  print("\nmotion %s %s: %d of %d ReLU pre-activations within %.1e of their scale of 0" %
        (case, prec, near, sum(v[1] for v in stats.values()), tsr.RELU_NEAR))
  _check("motion", case, prec, got, ref)

