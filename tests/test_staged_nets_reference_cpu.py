"""The float64 reference of the staged inference forward (train_stage_ref.make_forward_case / forward) on the CPU:
in mode "exact" it is the oracle's forward, a window of rays evaluated alone equals the same rays of the whole
call, and every planted error would fail tests/test_staged_nets_gpu.py's comparison of raw by a wide margin at a
reduced shape, so that its bars are not vacuous."""

import pytest
import torch

import train_stage_ref as tsr
from oracle import dynibar_oracle as orc

MARGIN = 3.0  # a planted error must exceed the GPU test's bf16 bar of raw (the larger of the two) by this factor


@pytest.fixture
def oracle_fp64(monkeypatch):
  """The oracle embeds the time of the dynamic net as `t.float()`; evaluate that embedding in float64 as well."""
  pe = orc.periodic_embed
  monkeypatch.setattr(orc, "periodic_embed", lambda x, n, linspace=False: pe(x.double(), n, linspace))


def _oracle(c):
  d = lambda x: x.double()
  w = {k: d(p.detach()) for k, p in c["mod"].named_parameters()}
  with torch.no_grad():
    if c["kind"] == "dynamic":
      return orc.net_dynamic(w, d(c["pts"]), d(c["feat"]), d(c["ray_dir"]), d(c["mask"]),
                             torch.tensor(c["t"], dtype=torch.float64), float(c["mod"].shift))
    return orc.net_static(w, d(c["pts"]), d(c["ref_rays"]), d(c["src_rays"]), d(c["feat"]), d(c["ray_diff"]),
                          d(c["mask"]), anti_alias_pooling=c["aa"], mask_rgb=c["mrgb"])


_EXACT_CASES = [
    ("dynamic", 3, 5, 20, False, False, True, False),
    ("dynamic", 4, 1, 17, False, False, False, False),
    ("static", 3, 5, 20, True, True, False, True),
    ("static", 2, 3, 32, True, True, True, False),
    ("static", 5, 2, 17, False, True, False, False),
]


@pytest.mark.parametrize("kind,R,S,V,aa,mrgb,hot,s_zero", _EXACT_CASES)
def test_exact_forward_is_the_oracle(oracle_fp64, kind, R, S, V, aa, mrgb, hot, s_zero):
  """Over V > 16, S = 1, hot weights, s = 0 and exactly black colours under mask_rgb, the reference's exact forward
  equals the oracle's in float64, and the cases hold what they promise."""
  c = tsr.make_forward_case(kind, R, S, V, aa, mrgb, hot, s_zero, seed=R + S + V)
  got, want = tsr.forward(c, "cpu", "exact"), _oracle(c)
  assert got.shape == want.shape == (R, S, 4)
  err = (got - want).abs().max().item()
  assert err <= 1e-10 * max(1.0, want.abs().max().item()), err
  nv = c["mask"].sum(2).flatten()
  assert (nv == 0).any() and (nv == 1).any() and (nv == V).any()
  assert (got[..., 3] == -1e9).any()
  if mrgb:
    assert (c["feat"][..., :3].sum(-1) == 0).any()


def test_hot_weights_leave_the_linear_range(monkeypatch):
  """The hot scale drives the visibility sigmoid into saturation for a fair share of (point, view) rows."""
  seen, frac = {}, {}
  lin = tsr._Net.lin

  def spy(self, name, segs, act, **kw):
    seen[name] = lin(self, name, segs, act, **kw)
    return seen[name]

  monkeypatch.setattr(tsr._Net, "lin", spy)
  for hot in (False, True):
    tsr.forward(tsr.make_forward_case("static", 4, 4, 20, True, False, hot, seed=9), "cpu", "exact")
    s = seen["vis_fc2.2"]
    frac[hot] = float(((s < 0.01) | (s > 0.99)).double().mean())
  assert frac[False] < 0.05 and frac[True] > 0.25, frac


def test_window_equals_the_same_rays_of_the_whole_call():
  """Rays are independent: a window evaluated alone gives the same raw as those rays of the whole evaluation (the
  GPU test compares windows of a chunked call with the reference evaluated on the window)."""
  c = tsr.make_forward_case("static", 9, 4, 18, True, True, seed=2)
  whole = tsr.forward(c, "cpu", "exact")
  for lo, hi in ((0, 3), (3, 7), (8, 9)):
    torch.testing.assert_close(tsr.forward(c, "cpu", "exact", lo, hi), whole[lo:hi], rtol=1e-12, atol=1e-12)


# plant -> (nets, R, S, V, rays [lo, hi) compared); rays_chunk0 with internal chunks of 4 rays
_PLANT_CASES = {
    "pool2_first16": (("dynamic", "static"), 4, 4, 32, None),
    "keys_first256": (("dynamic", "static"), 1, 384, 2, None),
    "rays_chunk0": (("dynamic", "static"), 8, 2, 3, (4, 8)),
    "blend_first16": (("static",), 2, 4, 20, None),
}


@pytest.mark.parametrize("plant,kind", [(p, k) for p, spec in _PLANT_CASES.items() for k in spec[0]])
def test_planted_error_exceeds_gpu_bar(plant, kind):
  kinds, R, S, V, rays = _PLANT_CASES[plant]
  lo, hi = rays if rays else (0, R)
  c = tsr.make_forward_case(kind, R, S, V, aa=kind == "static", mrgb=kind == "static", seed=3)
  ref = tsr.forward(c, "cpu", "kernel", lo, hi)
  got = tsr.forward(c, "cpu", "kernel", lo, hi, plant=plant, rays_per_chunk=4)
  r, errs = tsr.fwd_ratio(kind, "bf16", got, ref)
  print("\n%s %s: %.1fx the bf16 bar of raw (%.2e %.2e)" % (plant, kind, r, *errs))
  assert r >= MARGIN, (plant, kind, r, errs)
