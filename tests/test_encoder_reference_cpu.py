"""The float64 reference of the 2-D encoder's training forward and backward (tests/encoder_ref.py) on the CPU: in mode
"exact" it is torch autograd through oracle.encoder_forward, its bf16 emulation stays within a few bf16 ulps of the
exact evaluation, dispatch() makes the row and chunk decisions the GPU cases are chosen to cross, and every planted
wiring error would fail the GPU comparison (tests/test_encoder_train_gpu.py) by a wide margin, so that test's bars
are not vacuous."""

import pytest
import torch

import encoder_ref as er
from oracle import dynibar_oracle as orc

MARGIN = 3.0  # a planted error must exceed the GPU test's bf16 bar by this factor on some compared tensor


def _oracle(c):
  """torch autograd through oracle.encoder_forward in float64."""
  w = {k: v.double().clone().requires_grad_(True) for k, v in er.executed_params(c["mod"]).items()}
  co, fi = orc.encoder_forward(w, c["x"].double())
  loss = 0.0
  if c["gc"] is not None:
    loss = loss + (co * c["gc"].double()).sum()
  if c["gf"] is not None:
    loss = loss + (fi * c["gf"].double()).sum()
  loss.backward()
  res = {"coarse": co.detach(), "fine": fi.detach()}
  res.update({k: v.grad for k, v in w.items()})
  return res


@pytest.mark.parametrize("case", ["minimum", "small_odd", "mixed"])
def test_exact_mode_is_oracle_autograd(case):
  """Coarse, fine and every parameter gradient equal autograd through the oracle in float64, on 2-wide planes
  under reflect padding and odd sizes under stride 2.  (Not on case "flat": there even two float64 evaluations
  disagree, see tests/test_encoder_train_gpu.py.)"""
  c = er.make_case(case)
  got, want = er.reference(c, "cpu", "exact"), _oracle(c)
  assert set(got) == set(want)
  for k, b in want.items():
    err = (got[k] - b).abs().max().item()
    assert err <= 1e-10 * max(1.0, b.abs().max().item()), (k, err)


def test_exact_mode_one_output_gradient():
  """A gradient on one output only (bench.py trains coarse; the backward gets d fine = 0)."""
  c = er.make_case("small_odd")
  for drop in ("gc", "gf"):
    cc = dict(c, **{drop: None})
    got, want = er.reference(cc, "cpu", "exact"), _oracle(cc)
    for k, b in want.items():
      assert (got[k] - b).abs().max().item() <= 1e-10 * max(1.0, b.abs().max().item()), (drop, k)


def test_kernel_mode_agrees_with_exact_mode():
  """Rounding the tensor-core operands to bf16 (relative error <= 2^-9 each) moves every gradient by a few bf16 ulps
  of its scale in the L2 norm, and it does round.  Case at_2048: every product on the tensor cores; the forward and
  out_conv's bias (a column sum of dYt, fp32 SIMT) do not round."""
  c = er.make_case("at_2048")
  k, e = er.reference(c, "cpu", "kernel"), er.reference(c, "cpu", "exact")
  moved = 0
  for name, (rel, mx) in er.errors(k, e).items():
    assert rel <= 8 * 2 ** -9, (name, rel)
    moved += rel > 0
  for name in ("coarse", "fine", "out_conv.bias"):
    assert k[name].equal(e[name]), name
  assert moved == len(e) - 3, moved


def test_dispatch_rules():
  """The row threshold and the 256-column chunks the GPU cases are chosen to cross: stem K = 147, 3x3 K = 576,
  1x1 K = 64; rows N H2 W2 (stem) and N H4 W4 (layer1, out_conv)."""
  d = er.dispatch
  assert d("bf16", 2047, 576) == [(0, 256, False), (256, 512, False), (512, 576, False)]
  assert d("bf16", 2048, 576) == [(0, 256, True), (256, 512, True), (512, 576, True)]
  assert d("bf16", 2048, 147) == [(0, 147, True)]
  assert d("bf16", 10 ** 6, 64) == [(0, 64, True)]
  assert d("fp32", 10 ** 6, 576) == [(0, 256, False), (256, 512, False), (512, 576, False)]
  rows = {}
  for name, (N, H, W, _) in er.CASES.items():
    H2, W2, H4, W4 = er.dims(H, W)
    rows[name] = (N * H2 * W2, N * H4 * W4)
  assert rows == {"minimum": (16, 4), "small_odd": (459, 135), "mixed": (3456, 864), "below_2048": (7965, 2047),
                  "at_2048": (8192, 2048), "ragged": (23175, 5928), "flat": (3072, 768),
                  "bench": (294912, 73728)}
  tc = {n: (d("bf16", a, 147)[0][2], d("bf16", b, 576)[0][2]) for n, (a, b) in rows.items()}
  assert tc["minimum"] == tc["small_odd"] == (False, False)
  assert tc["mixed"] == tc["below_2048"] == tc["flat"] == (True, False)
  assert tc["at_2048"] == tc["ragged"] == tc["bench"] == (True, True)
  assert rows["ragged"][0] % 128 == 7 and rows["ragged"][1] % 128 == 40  # partial last tiles at both resolutions


def test_im2col_col2im_are_adjoint():
  """<im2col(X), C> = <X, col2im(C)> for the reflect map, the zero-padding map differs (what the plant
  col2im_zero_pad breaks), and im2col equals unfold of the reflect-padded input."""
  g = torch.Generator().manual_seed(0)
  for (H, W, k, s, p) in [(9, 13, 3, 2, 1), (4, 4, 7, 2, 3), (2, 2, 3, 1, 1), (6, 5, 1, 2, 0)]:
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    X = torch.randn(2, 3, H, W, generator=g, dtype=torch.float64)
    C = torch.randn(2 * Ho * Wo, 3 * k * k, generator=g, dtype=torch.float64)
    lhs = (er.im2col(X, k, s, p, Ho, Wo) * C).sum()
    rhs = (X * er.col2im(C, X.shape, k, s, p, Ho, Wo)).sum()
    assert abs(float(lhs - rhs)) <= 1e-12 * float(C.abs().sum()), (H, W, k)
    Xp = torch.nn.functional.pad(X, (p,) * 4, mode="reflect") if p else X
    u = torch.nn.functional.unfold(Xp, k, stride=s).transpose(1, 2).reshape(-1, 3 * k * k)
    assert torch.equal(er.im2col(X, k, s, p, Ho, Wo), u)
    if p:
      assert not torch.allclose(er.col2im(C, X.shape, k, s, p, Ho, Wo, zero_pad=True),
                                er.col2im(C, X.shape, k, s, p, Ho, Wo))


# plant -> the case it is scored on (a case of the GPU test where the wiring it breaks runs on the tensor cores)
_PLANT_CASES = {
    "dw_ragged_tile": "ragged",
    "in_drop_xh_term": "ragged",
    "col2im_zero_pad": "ragged",
    "dx_drop_last_chunk": "ragged",
    "b0_im2col_pad0": "ragged",
    "bn_swap": "ragged",
    "d_fine_ignored": "ragged",
    "ds_dx_overwrite": "ragged",
}

_cache = {}


def _margin(plant):
  name = _PLANT_CASES[plant]
  if name not in _cache:
    c = er.make_case(name)
    _cache[name] = (c, er.reference(c, "cpu", "kernel"))
  c, ref = _cache[name]
  got = er.reference(c, "cpu", "kernel", plant=plant)
  r = er.ratios("bf16", got, ref)
  return max(r.values()), r


@pytest.mark.parametrize("plant", er.PLANTS)
def test_planted_error_exceeds_gpu_bar(plant):
  m, r = _margin(plant)
  assert m >= MARGIN, (plant, sorted(r.items(), key=lambda kv: -kv[1])[:4])


def test_smallest_plant_margin(capsys):
  margins = {p: _margin(p) for p in er.PLANTS}
  with capsys.disabled():
    for p, (m, r) in margins.items():
      print("\nplanted %s: %.1fx the bf16 bar (%s)" % (p, m, max(r, key=r.get)), end="")
    p, (m, _) = min(margins.items(), key=lambda kv: kv[1][0])
    print("\nsmallest planted-error margin: %.1fx (%s)" % (m, p))
  assert m >= MARGIN
