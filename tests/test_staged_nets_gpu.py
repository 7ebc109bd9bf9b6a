"""The staged evaluation of DynibarDynamic and DynibarStatic (csrc/nets_f32.cu: net_dynamic_f32 / net_static_f32)
against the float64 reference of tests/train_stage_ref.py, past the shapes of tests/test_train_stage_gpu.py:
17-32 source views, 1 to 384 samples per ray, several internal chunks.

The inference forward (render_ray.net_dynamic_forward / net_static_forward, the staged path of every fp32 render and
of every bf16 render with more than 16 views) is compared in precision "fp32" with the reference in mode "exact"
and in precision "bf16" with mode "kernel", which rounds the operands of exactly the products run_lin puts on the
tensor cores (M >= 128 rows and >= 16 outputs; train_stage_ref.dispatch).  raw is compared in full, the -1e9
sigma of a point no view sees exactly.  The inputs hold points with 0, 1 and all views valid, exactly black source
colours under mask_rgb, anti-aliased pooling with s = 0, and "hot" weights (train_stage_ref.make_forward_case).

  v17 .. v32   the kMaxViews-sized per-thread arrays of st_pool1, pool2 and st_out; v32_r128 puts every layer of
               the bf16 path on the tensor cores, the per-ray ref_feature_fc included
  s1, s2       attention over one and two samples
  s192 .. s384 the SIMT attention at its 48 KiB shared-memory boundary (S = 192), past it (the opt-in attribute),
               and at S = 384
  dyn_vv       the dynamic net at 29 + 3 virtual views, the V the monocular path passes
  chunks       R = 2 * 8192 + 3 rays of S = 16, V = 32: three internal chunks (net_rows_per_chunk = 8192).  The
               second chunk and the 3-ray tail must equal, bit for bit, separate calls on just those rays (the
               rays are independent, and a call of one chunk's rays takes that chunk's dispatch).  128-ray windows
               at the start, across the chunk-0/1 boundary and at the end of chunk 1, and the whole tail, are
               compared with the reference evaluated on the window alone: a window of >= 128 rays has a full
               chunk's dispatch, and the tail (P = 48 < 128) runs its per-point layers and ref_feature_fc in SIMT
               in both.  The library's workspace is 11.7 GiB (dynamic) / 20.6 GiB (static) for the one chunk it
               holds at a time; the inputs add 1.6 GB.

The training forward and backward (autograd.net_dynamic / net_static) are compared like
tests/test_train_stage_gpu.py, every output and gradient, at V = 17 and 32 and S = 128 to 384.  S above 288 runs the
attention backward's bounded instance (attention_bwd_wide_kernel); S = 385 is refused before any forward work.

Bars, measured on an H100 80GB HBM3 (700 W) and set as in tests/test_train_stage_gpu.py (2x the worst, rounded up to
one digit):
  - raw of the cases with ordinary weights stays within the training comparison's bar of raw
    (train_stage_ref.FWD_BARS = BARS[...]["out"]), at most 0.5 of it, chunk windows and tail included.
  - The hot cases (v24, s2, s193) have their own bars (train_stage_ref.FWD_HOT_BARS).  Scaling every weight by 4
    compounds over a dozen layers: fp32 drifts to 2e-5 of the float64 value, as much as the same reference evaluated
    in float32 on the CPU.  The static blending logits reach a few hundred, so the softmax over views is nearly an
    argmax.  A bf16 rounding of a logit then hands a near-tie to the other view, and a few such points move raw by
    up to 0.29 of its largest value (static s193, bf16).  The hot bf16 static bar is therefore loose.  The tight
    bars of the other cases are the ones that catch wiring errors.
  - The training cases use train_stage_ref.BARS, except where TRAIN_BARS states a measured bar.
tests/test_staged_nets_reference_cpu.py shows each planted error of train_stage_ref.FWD_PLANTS exceeds the bf16 bar
of raw at least 3x.  Three errors planted in the kernels were each caught: the chunk's ray offset dropped from
ray_dir / ref_rays, st_out_kernel's loops capped at 16 views, and pool2_kernel's loops capped at 16 views.  The file
runs in about 12 s on one H100 (26 s with interpreter start-up).
"""

import pytest
import torch

import train_stage_ref as tsr
from test_train_stage_gpu import _library as _train_library

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# name: (nets, R, S, V, anti_alias, mask_rgb, hot, s_zero); anti_alias / mask_rgb / s_zero apply to the static net
FWD_CASES = {
    "v17": (("dynamic", "static"), 6, 16, 17, True, True, False, False),
    "v24": (("dynamic", "static"), 5, 16, 24, True, False, True, False),
    "v31": (("dynamic", "static"), 4, 16, 31, True, True, False, True),
    "v32": (("dynamic", "static"), 3, 16, 32, False, True, False, False),
    "v32_r128": (("dynamic", "static"), 128, 16, 32, True, True, False, False),
    "s1": (("dynamic", "static"), 40, 1, 20, True, False, False, False),
    "s2": (("dynamic", "static"), 40, 2, 20, False, True, True, False),
    "s192": (("dynamic", "static"), 2, 192, 17, True, False, False, False),
    "s193": (("dynamic", "static"), 2, 193, 17, True, True, True, False),
    "s384": (("dynamic", "static"), 1, 384, 17, True, False, False, False),
    "dyn_vv": (("dynamic",), 8, 16, 29 + 3, False, False, False, False),
}
CHUNK_RAYS = 8192  # net_rows_per_chunk(16, 32) = 4194304 / (16 * 32)

# name: (R, S, V, anti_alias, mask_rgb), as train_stage_ref.NET_CASES
TRAIN_CASES = {
    "v17": (64, 16, 17, True, True),
    "v32": (32, 16, 32, True, False),
    "s128": (16, 128, 4, True, False),
    "s192": (8, 192, 3, False, True),
    "s288": (4, 288, 3, True, False),
    "s320": (4, 320, 3, True, True),
    "s384": (3, 384, 5, True, False),
}


def _device_module(c):
  if "dev_mod" not in c:
    import copy
    c["dev_mod"] = copy.deepcopy(c["mod"]).to(DEV).requires_grad_(False)
  return c["dev_mod"]


def _forward(c, prec, lo=0, hi=None):
  """The library's inference forward of rays [lo, hi) in precision `prec`."""
  from dynibar_b200 import render_ray as rr
  mod = _device_module(c)
  hi = c["feat"].shape[0] if hi is None else hi
  d = lambda k: c[k][lo:hi].to(DEV)
  with torch.no_grad(), rr.precision_scope(prec):
    if c["kind"] == "dynamic":
      out = rr.net_dynamic_forward(mod, d("pts"), d("feat"), d("ray_dir"), d("mask"), c["t"])
    else:
      out = rr.net_static_forward(mod, d("pts"), d("ref_rays"), d("src_rays"), d("feat"), d("ray_diff"), d("mask"))
  torch.cuda.synchronize()
  return out


def _check_fwd(kind, case, prec, got, ref, hot=False):
  r, (rel, mx) = tsr.fwd_ratio(kind, prec, got, ref, hot)
  print("\n  FWD %s %s %s %.3e %.3e (%.2f of its bar)" % (kind, case, prec, rel, mx, r))
  assert torch.isfinite(got).all(), (kind, case, prec)
  assert r <= 1.0, (kind, case, prec, rel, mx)


# Training bars that the cases here need above train_stage_ref.BARS: (net, precision, tensor) -> bar; the comment
# records the measured worst and its case.
TRAIN_BARS = {
    ("dynamic", "bf16", "rgb_fc.2.bias"): (2e-03, 2e-03),  # 5.04e-04 s128, 9.27e-04 s384
    ("static", "fp32", "out"): (1e-05, 8e-05),  # 1.17e-06 3.84e-05 s288
}


def _check_train(kind, case, prec, got, ref, V):
  errs = tsr.errors(kind, got, ref, V)
  bar = lambda k: TRAIN_BARS.get((kind, prec, k), tsr.bar(kind, prec, k))
  r = {k: max(rel / bar(k)[0], mx / bar(k)[1]) for k, (rel, mx) in errs.items()}
  print("\n%s %s %s: worst %s, %.2f of its bar" % (kind, case, prec, *max(r.items(), key=lambda kv: kv[1])))
  for name, (rel, mx) in sorted(errs.items()):
    print("  ERR %s %s %s %s %.3e %.3e" % (kind, case, prec, name, rel, mx))
  bad = {k: (errs[k], bar(k)) for k, v in r.items() if not v <= 1.0}
  assert not bad, (kind, case, prec, bad)


def _mode(prec):
  return "kernel" if prec == "bf16" else "exact"


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("kind,case", [(k, n) for n, spec in FWD_CASES.items() for k in spec[0]])
def test_inference_forward_matches_reference(kind, case, prec):
  _, R, S, V, aa, mrgb, hot, s_zero = FWD_CASES[case]
  static = kind == "static"
  c = tsr.make_forward_case(kind, R, S, V, aa and static, mrgb and static, hot, s_zero and static,
                            seed=R + S + V, device=DEV)
  got = _forward(c, prec)
  ref = tsr.forward(c, DEV, _mode(prec))
  assert bool((ref[..., 3] == -1e9).any())  # the sentinel is exercised
  _check_fwd(kind, case, prec, got, ref, hot)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("kind", ["dynamic", "static"])
def test_inference_forward_across_internal_chunks(kind, prec):
  from dynibar_b200 import _lib
  S, V, RC = 16, 32, CHUNK_RAYS
  R = 2 * RC + 3
  code = _lib.NET_DYNAMIC if kind == "dynamic" else _lib.NET_STATIC
  ws = lambda r: int(_lib.lib.dyn_net_workspace_bytes(code, r, S, V))
  assert ws(RC - 1) < ws(RC) == ws(R)  # the workspace holds exactly one chunk of RC rays
  c = tsr.make_forward_case(kind, R, S, V, aa=kind == "static", mrgb=kind == "static", seed=5, device=DEV)
  full = _forward(c, prec)
  assert torch.equal(full[RC:2 * RC], _forward(c, prec, RC, 2 * RC))
  assert torch.equal(full[2 * RC:], _forward(c, prec, 2 * RC, R))
  for lo, hi in ((0, 128), (RC - 64, RC + 64), (2 * RC - 128, 2 * RC), (2 * RC, R)):
    ref = tsr.forward(c, DEV, _mode(prec), lo, hi)
    _check_fwd(kind, "chunks[%d:%d]" % (lo, hi), prec, full[lo:hi], ref)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("case", list(TRAIN_CASES))
@pytest.mark.parametrize("kind", ["dynamic", "static"])
def test_training_matches_reference(kind, case, prec):
  R, S, V, aa, mrgb = TRAIN_CASES[case]
  c = tsr.make_net_case(kind, R, S, V, aa, mrgb, seed=R + S + V)
  got = _train_library(c, prec)
  ref = tsr.reference(c, DEV, _mode(prec))
  _check_train(kind, case, prec, got, ref, V)


@pytest.mark.parametrize("kind", ["dynamic", "static"])
def test_training_refuses_samples_past_the_attention_backward_limit(kind):
  """S = 385 passes the inference forward's attention limit but not the backward's; the training forward refuses
  it at entry, naming the limit."""
  c = tsr.make_net_case(kind, 1, 385, 2, seed=7)
  with pytest.raises(RuntimeError, match=r"attention backward supports S <= 384 samples per ray \(got 385\)"):
    _train_library(c, "fp32")
