"""The criterion without a GPU: the torch restatement (tests/loss_ref.py) against the reference's own helpers
(tests/golden/loss_terms.pt) and against the definition of the distortion loss, and the host side of
dynibar_b200.criterion (the weight struct of an epoch; CPU tensors are refused)."""

import math
import os
import sys
from types import SimpleNamespace

import pytest
import torch

import loss_ref

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden_loss as mgl  # noqa: E402

TOL = dict(rtol=2e-4, atol=2e-5)  # the bar of test_oracle_golden.py


def _args(**kw):
  a = dict(w_disp=5e-2, w_flow=5e-3, w_cycle=0.1, cycle_factor=0.1, anneal_cycle=False, w_reg=0.05,
           w_skew_entropy=1e-3, w_distortion=1e-3, decay_rate=10.0, init_decay_epoch=150)
  a.update(kw)
  return SimpleNamespace(**a)


@pytest.mark.parametrize("case", list(mgl.CASES))
def test_helper_terms_match_the_reference(case, golden):
  fx = golden("loss_terms")[case]
  x = mgl.inputs(**mgl.CASES[case])
  o, rb, mm = x["outputs"], x["ray_batch"], x["motion_mask"]
  got_sum = float(sum(v.double().sum() for v in (o["rgb"], rb["rgb"], x["render_flow"], x["pred_mask"])))
  assert abs(got_sum - fx["input_sum"]) < 1e-9 * abs(fx["input_sum"]), "seeded inputs drifted from the fixture's"
  got = {"criterion": loss_ref.criterion_rgb(o, rb), "criterion_motion": loss_ref.criterion_rgb(o, rb, mm),
         "rgb": loss_ref.rgb_loss(o["rgb"], rb, x["pred_mask"]),
         "temporal": loss_ref.temporal_rgb(o, rb), "temporal_motion": loss_ref.temporal_rgb(o, rb, mm),
         "flow": loss_ref.flow_l1(x["render_flow"], x["gt_flow"], x["flow_mask"])}
  for k, v in got.items():
    torch.testing.assert_close(v, fx[k], msg=lambda m: k + ": " + m, **TOL)


@pytest.mark.parametrize("R,S,seed", [(7, 63, 1), (3, 5, 2), (2, 1, 3)])
def test_distortion_prefix_sum_form_equals_its_definition(R, S, seed):
  g = torch.Generator().manual_seed(seed)
  s = torch.sort(torch.rand(R, S + 1, generator=g, dtype=torch.float64), dim=1).values
  w = torch.rand(R, S, generator=g, dtype=torch.float64)
  m, iv = (s[:, 1:] + s[:, :-1]) * 0.5, s[:, 1:] - s[:, :-1]
  torch.testing.assert_close(loss_ref.distortion(w, m, iv), loss_ref.distortion_pairwise(w, m, iv), rtol=1e-10,
                             atol=0.0)


# (epoch, overrides) -> what train.py:302-357 gives
@pytest.mark.parametrize("epoch,kw", [(0, {}), (149, {}), (150, {}), (449, {}), (750, {}), (900, dict(decay_rate=2.0)),
                                       (300, dict(anneal_cycle=True)), (900, dict(anneal_cycle=True)),
                                       (450, dict(anneal_cycle=True, w_cycle=0.3, cycle_factor=0.05)),
                                       (20, dict(init_decay_epoch=10, anneal_cycle=True))])
def test_step_weights_follow_the_epoch(epoch, kw):
  from dynibar_b200 import criterion as cr
  args = _args(**kw)
  wt = cr.step_weights(args, epoch)
  divisor = epoch // args.init_decay_epoch
  on = lambda k: bool((wt.terms >> k) & 1)
  close = lambda a, b: math.isclose(a, b, rel_tol=1e-6)
  assert on(cr.RGB_DYNAMIC) == (epoch < args.init_decay_epoch)
  assert on(cr.STATIC_DY) == (divisor > 4)
  always = (cr.RGB_REF, cr.RGB_ANCHOR, cr.RGB_REF_DY, cr.RGB_ANCHOR_DY, cr.STATIC, cr.DISP, cr.FLOW, cr.CYCLE,
            cr.REG_ABS, cr.REG_TIME, cr.REG_SPACE, cr.ENTROPY, cr.DISTORTION)
  assert all(on(k) for k in always) and wt.terms >> 15 == 0
  assert wt.w[cr.RGB_REF] == wt.w[cr.RGB_ANCHOR] == wt.w[cr.STATIC] == 1.0
  assert close(wt.w[cr.RGB_REF_DY], 1.0 / 10.0 ** divisor) and close(wt.w[cr.RGB_ANCHOR_DY], 1.0 / 10.0 ** divisor)
  assert close(wt.w[cr.DISP], args.w_disp / args.decay_rate ** divisor)
  assert close(wt.w[cr.FLOW], args.w_flow / args.decay_rate ** divisor)
  want_cycle = min(0.5, args.w_cycle + divisor * args.cycle_factor) if args.anneal_cycle else args.w_cycle
  assert close(wt.w[cr.CYCLE], want_cycle)
  assert close(wt.w[cr.REG_ABS], args.w_reg) and close(wt.w[cr.REG_TIME], 0.5 * args.w_reg)
  assert close(wt.w[cr.REG_SPACE], args.w_reg)
  assert close(wt.w[cr.ENTROPY], args.w_skew_entropy) and close(wt.w[cr.DISTORTION], args.w_distortion)
  if on(cr.STATIC_DY):
    assert close(wt.w[cr.STATIC_DY], 0.1)
  assert [close(e, 1e-8 if k in (cr.RGB_ANCHOR, cr.RGB_ANCHOR_DY) else 1e-6) for k, e in enumerate(wt.rgb_eps)] == \
      [True] * 6
  # and the restatement the GPU tests compare against agrees
  sw = loss_ref.step_weights(args, epoch)
  assert close(sw["w_cycle"], wt.w[cr.CYCLE]) and close(sw["w_disp"], wt.w[cr.DISP])
  assert sw["dynamic_rgb"] == on(cr.RGB_DYNAMIC) and sw["static_dy"] == on(cr.STATIC_DY)


def test_anneal_cycle_is_capped_at_one_half():
  from dynibar_b200 import criterion as cr
  assert cr.step_weights(_args(anneal_cycle=True), 150 * 3).w[cr.CYCLE] == pytest.approx(0.4)
  assert cr.step_weights(_args(anneal_cycle=True), 150 * 4).w[cr.CYCLE] == pytest.approx(0.5)
  assert cr.step_weights(_args(anneal_cycle=True), 150 * 9).w[cr.CYCLE] == pytest.approx(0.5)
  assert cr.step_weights(_args(anneal_cycle=False), 150 * 9).w[cr.CYCLE] == pytest.approx(0.1)


def _fake_step(R=6, S=8, K=2):
  g = torch.Generator().manual_seed(0)
  rnd = lambda *s: torch.rand(*s, generator=g)
  comp = lambda: {"rgb": rnd(R, 3), "mask": rnd(R) > 0.2, "weights": rnd(R, S)}
  ref = dict(comp(), rgb_dy=rnd(R, 3), rgb_static=rnd(R, 3), depth=rnd(R) * 5, weights_dy=rnd(R, S),
             weights_st=rnd(R, S), render_flows=rnd(6, R, 2), s_vals=torch.sort(rnd(R, S), dim=1).values)
  anc = dict(comp(), occ_weights=rnd(R, S), occ_weight_map=rnd(R), pts_traj_ref=rnd(K, R, S, 3),
             pts_traj_anchor=rnd(K, R, S, 3), sf_seq=rnd(6, R, S, 3))
  ret = {"outputs_coarse_ref": ref, "outputs_coarse_ref_dy": comp(), "outputs_coarse_st": comp(),
         "outputs_coarse_anchor": anc, "outputs_coarse_anchor_dy": dict(comp(), occ_weight_map=rnd(R))}
  rb = {"rgb": rnd(R, 3), "disp": rnd(R), "motion_mask": (rnd(R) > 0.5).float(), "flows": rnd(6, R, 2),
        "masks": (rnd(6, R, 1) > 0.3).float()}
  rb["static_mask"] = 1.0 - rb["motion_mask"]
  return ret, rb


def test_cpu_tensors_are_refused():
  from dynibar_b200 import criterion as cr
  ret, rb = _fake_step()
  with pytest.raises(RuntimeError, match="no CPU fallback"):
    cr.mono_step_loss(ret, rb, _args(), 0)
  with pytest.raises(RuntimeError, match="no CPU fallback"):
    cr.static_bootstrap_loss(ret, rb)
  with pytest.raises(RuntimeError, match="no CPU fallback"):
    cr.compute_flow_loss(rb["flows"], rb["flows"], rb["masks"])
  # the restatement runs on the same dicts, in float64 too
  loss, terms = loss_ref.mono_step_loss(ret, rb, _args(), 900)
  assert torch.isfinite(loss) and set(terms) == set(cr.TERM_NAMES)
