"""The float64 reference of the training forward and backward (tests/train_stage_ref.py) on the CPU: in mode "exact"
it is torch autograd through the oracle, its bf16 emulation stays within a few bf16 ulps of the exact evaluation,
and every planted wiring error would fail the GPU comparison (tests/test_train_stage_gpu.py) by a wide margin, so
that test's bars are not vacuous."""

import pytest
import torch

import train_stage_ref as tsr
from oracle import dynibar_oracle as orc

MARGIN = 3.0  # a planted error must exceed the GPU test's bar by this factor on some compared tensor


def _oracle(c):
  """torch autograd through the oracle in float64, every gradient the library returns."""
  d = lambda x: x.double()
  w = {k: d(p.detach()).requires_grad_(True) for k, p in c["mod"].named_parameters()}
  if c["kind"] == "motion":
    x = d(c["xyzt"]).requires_grad_(True)
    out, ins = orc.motion_mlp(w, x), {"xyzt": x}
  elif c["kind"] == "dynamic":
    pts, feat = d(c["pts"]).requires_grad_(True), d(c["feat"]).requires_grad_(True)
    out = orc.net_dynamic(w, pts, feat, d(c["ray_dir"]), d(c["mask"]), torch.tensor(c["t"], dtype=torch.float64),
                          float(c["mod"].shift))
    ins = {"pts": pts, "rgb_feat": feat}
  else:
    feat = d(c["feat"]).requires_grad_(True)
    out = orc.net_static(w, d(c["pts"]), d(c["ref_rays"]), d(c["src_rays"]), feat, d(c["ray_diff"]), d(c["mask"]),
                         anti_alias_pooling=c["aa"], mask_rgb=c["mrgb"])
    ins = {"rgb_feat": feat}
  (out * d(c["gen"])).sum().backward()
  res = {"out": out.detach()}
  res.update({k: v.grad for k, v in w.items()})
  res.update({k: v.grad for k, v in ins.items()})
  return res


@pytest.fixture
def oracle_fp64(monkeypatch):
  """The oracle embeds the time of the dynamic net as `t.float()`; evaluate that embedding in float64 as well."""
  pe = orc.periodic_embed
  monkeypatch.setattr(orc, "periodic_embed", lambda x, n, linspace=False: pe(x.double(), n, linspace))
  return _oracle


_EXACT_CASES = [
    ("dynamic", 3, 16, 5, False, False),
    ("dynamic", 2, 8, 1, False, False),
    ("static", 3, 16, 5, True, False),
    ("static", 3, 8, 4, False, True),
    ("static", 2, 8, 3, True, True),
]


@pytest.mark.parametrize("kind,R,S,V,aa,mrgb", _EXACT_CASES)
def test_exact_mode_is_oracle_autograd(oracle_fp64, kind, R, S, V, aa, mrgb):
  """Every output and gradient equals autograd through oracle.net_dynamic / net_static in float64.  The cases
  cover anti-alias pooling on and off, mask_rgb, points with 0, 1 and all views valid (the query-row mask of the
  ray transformer), and V = 1."""
  c = tsr.make_net_case(kind, R, S, V, aa, mrgb, seed=R + S + V)
  got, want = tsr.reference(c, "cpu", "exact"), oracle_fp64(c)
  assert set(got) == set(want)
  for k, b in want.items():
    err = (got[k] - b).abs().max().item()
    assert err <= 1e-10 * max(1.0, b.abs().max().item()), (k, err)
  nv = c["mask"].sum(2).flatten()
  assert (nv == 0).any() and (nv == 1).any() and (nv == V).any()


@pytest.mark.parametrize("nb", [4, 6])
def test_exact_mode_is_oracle_autograd_motion(oracle_fp64, nb):
  c = tsr.make_motion_case(300, nb, seed=nb)
  got, want = tsr.reference(c, "cpu", "exact"), oracle_fp64(c)
  assert set(got) == set(want)
  for k, b in want.items():
    err = (got[k] - b).abs().max().item()
    assert err <= 1e-10 * max(1.0, b.abs().max().item()), (k, err)


def _bf16_case(kind):
  # P = 2096 (not a multiple of 64): every per-point and per-view product is on the tensor cores
  if kind == "motion":
    return tsr.make_motion_case(2100, 6, seed=3)
  return tsr.make_net_case(kind, 131, 16, 3, aa=kind == "static", mrgb=kind == "static", seed=3)


@pytest.mark.parametrize("kind", ["dynamic", "static", "motion"])
def test_kernel_mode_agrees_with_exact_mode(kind):
  """Rounding the tensor-core operands to bf16 (relative error <= 2^-9 each) moves every gradient by a few bf16
  ulps of its scale in the L2 norm, and it does round.  Bias vectors are column sums whose terms cancel (the
  pooling weights are normalised), so their relative change is larger; the MotionMLP's ReLUs flip where bf16 moves
  a pre-activation across 0."""
  c = _bf16_case(kind)
  k, e = tsr.reference(c, "cpu", "kernel"), tsr.reference(c, "cpu", "exact")
  moved = 0
  for name, (rel, mx) in tsr.errors(kind, k, e).items():
    ulps = 128 if kind == "motion" else (16 if e[name].dim() > 1 else 64)
    assert rel <= ulps * 2 ** -9, (name, rel)
    moved += rel > 0
  assert moved >= len(e) // 2, moved


def test_dispatch_rules():
  """The thresholds the GPU cases are chosen to cross."""
  d = tsr.dispatch
  assert d("fwd", "dynamic", 128, 128, 127) == [(0, 128, False)]
  assert d("fwd", "dynamic", 3, 64, 10 ** 6) == [(0, 64, False)]
  assert d("fwd", "static", 16, 66, 128) == [(0, 66, True)]
  assert d("fwd", "motion", 256, 132, 128) == [(0, 132, True)]
  assert d("fwd", "motion", 18, 256, 10 ** 6, layer="coeff_linear") == [(0, 256, False)]
  assert d("grad_w", "dynamic", 256, 257, 2048) == [(0, 256, True), (256, 257, True)]
  assert d("grad_w", "dynamic", 256, 257, 2047) == [(0, 257, False)]
  assert d("grad_in", "dynamic", 256, 257, 2048) == [(0, 256, True), (256, 257, False)]
  assert d("grad_in", "dynamic", 128, 128, 10 ** 6, accumulate=True) == [(0, 128, False)]
  assert d("grad_in", "motion", 256, 388, 2048) == [(0, 256, True), (256, 388, True)]
  assert d("grad_in", "motion", 12, 256, 10 ** 6) == [(0, 256, False)]
  assert d("grad_in", "motion", 18, 256, 2048) == [(0, 256, True)]
  assert d("grad_w", "motion", 12, 256, 2048) == [(0, 256, True)]


# plant -> the case it is scored on (a case of the GPU test where the wiring it breaks is exercised)
_PLANT_CASES = {
    "rowscale_dw": ("static", "ragged"),
    "geo0_rem_col0": ("dynamic", "ragged"),
    "skip_dIn_drop": ("motion", "n2049"),
    "partial_stage": ("static", "ragged"),
    "bcast_one": ("dynamic", "v16"),
    "bias_P": ("static", "view_tc"),
    "acc_overwrite": ("dynamic", "view_tc"),
    "nblock_x": ("dynamic", "ragged"),
}


def _plant_case(kind, name):
  if kind == "motion":
    return tsr.make_motion_case(*tsr.MOTION_CASES[name], seed=1)
  R, S, V, aa, mrgb = tsr.NET_CASES[name]
  return tsr.make_net_case(kind, R, S, V, aa, mrgb, seed=1)


_cache = {}


def _margin(plant):
  kind, name = _PLANT_CASES[plant]
  c = _plant_case(kind, name)
  if (kind, name) not in _cache:
    _cache[(kind, name)] = tsr.reference(c, "cpu", "kernel")
  ref = _cache[(kind, name)]
  got = tsr.reference(c, "cpu", "kernel", plant=plant)
  r = tsr.ratios(kind, "bf16", got, ref, None if kind == "motion" else c["feat"].shape[2])
  return max(r.values()), r


@pytest.mark.parametrize("plant", tsr.PLANTS)
def test_planted_error_exceeds_gpu_bar(plant):
  m, r = _margin(plant)
  assert m >= MARGIN, (plant, sorted(r.items(), key=lambda kv: -kv[1])[:4])


def test_smallest_plant_margin(capsys):
  margins = {p: _margin(p)[0] for p in tsr.PLANTS}
  p, m = min(margins.items(), key=lambda kv: kv[1])
  with capsys.disabled():
    print("\nsmallest planted-error margin: %.1fx (%s)" % (m, p))
  assert m >= MARGIN
