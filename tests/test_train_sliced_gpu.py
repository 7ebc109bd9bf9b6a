"""A monocular training step in ray slices (dynibar_b200.train_step.mono_step_backward) on the device.

  1. The split criterion: rows of every slice plus one finish give the bits of dyn_mono_loss on the whole batch (all
     40 floats), and the slices' backward against the batch table gives the bits of the whole-batch backward (each
     element is written once, no atomics).  Generated inputs (test_loss_gpu.generated), all 15 terms on, R 1024 / 1000
     / 3072 in slice plans with a ragged last slice, K = 0 (cycle off) and the late epoch.
  2. The sliced step against the whole-batch step (train_step_ref's shipped / late / edges_occ1 cases, bf16 and fp32,
     the same jitter): loss, terms and every criterion input bit for bit; every gradient within SPREAD_BARS.
  3. The shipped batch: 3072 rays in slices of 1024, bf16, against train_step_ref.reference(mode="kernel") in float64
     evaluated in 128-ray chunks, within the bf16 bars of tests/test_train_step_gpu.py; the step's peak memory is printed.
  4. The static warm-up (bootstrap=True), sliced against whole, within SPREAD_BARS.
  5. A planted error: each slice normalised by its own denominators instead of the batch's misses SPREAD_BARS by at
     least train_step_ref.PLANT_MARGIN.

Measured on an H100 80GB HBM3 (700 W power limit, SM clock 1980 MHz): the loss, the nine terms and every criterion input
of the sliced step are bit-identical to the whole batch's in every case (no forward kernel's result depends on the
neighbouring rays).  The gradients are not: two whole-batch runs differ by up to 1.9e-6 relative L2 (the float atomics
of the network backward), a sliced step differs from the whole batch by up to 2.0e-5 (net_coarse_dy.base_fc.0.weight,
max-abs ratio) -- up to 110x that spread, and non-zero where it is 0 -- because slicing re-partitions every dW reduction over rows: each slice's
split-K slabs start at other rows, and the slices' sums add up in .grad.  So SPREAD_BARS are 2x the measured
sliced-vs-whole difference per tensor (the atomics spread is printed beside each), still far below the float64
reference's bars.  The 3072-ray batch sits at 0.49 of tests/test_train_step_gpu.py's bf16 bars (worst featmaps[1]),
which it therefore uses (SHIPPED_BARS).  The planted per-slice normalisation moves featmaps[2] by more than 1e5
times its bar.  Step peak memory at 3072 rays: 21.4 GB.
"""

import time

import pytest
import torch

import test_loss_gpu as TL
import train_step_ref as T
from dynibar_b200 import autograd as ag, criterion as cr, render_ray as rr, synthetic, train_step as ts
from dynibar_b200.projection import Projector

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODE = {"bf16": "kernel", "fp32": "exact"}
_AXIS1 = ("render_flows", "pts_traj_ref", "pts_traj_anchor", "sf_seq", "flows", "masks")

# ---------------------------------------------------------------------------------------------------------------
# 1. the split criterion
# ---------------------------------------------------------------------------------------------------------------
LATE = 5 * TL.INIT_DECAY + 1
SPLIT_CASES = [(1024, 3, 0, (512, 336)), (1000, 3, 0, (504, 336, 256)), (3072, 3, 0, (1024, 1000, 776)),
               (1000, 0, 0, (336,)), (1024, 3, LATE, (336,)), (3072, 3, LATE, (1000, 512))]


def _cut(d, lo, hi):
  return {k: (v[:, lo:hi] if k in _AXIS1 else v[lo:hi]) if torch.is_tensor(v) else v for k, v in d.items()}


def _criterion_call(ret, rb, args, epoch):
  """_step_call with every term that has inputs switched on (STATIC_DY and RGB_DYNAMIC together at epoch 0)."""
  wt, fixed, inputs = cr._step_call(ret, rb, args, epoch)
  if epoch == 0:
    wt.terms |= 1 << cr.STATIC_DY
    wt.w[cr.STATIC_DY] = 0.1
  return wt, fixed, inputs


def _leaves(ret):
  return {o: {k: v.detach().clone().requires_grad_(k in TL.GRAD_KEYS.get(o, ())) if v.is_floating_point() else v
              for k, v in d.items()} for o, d in ret.items()}


@pytest.mark.parametrize("R,K,epoch,sizes", SPLIT_CASES)
def test_split_criterion_gives_the_whole_batch_bits(R, K, epoch, sizes):
  ret, rb = TL.generated(R, 64, K, 4000 + R + K + epoch)
  ret = {o: {k: v.to(DEV) for k, v in d.items()} for o, d in ret.items()}
  rb = {k: v.to(DEV) for k, v in rb.items()}
  args = TL.loss_args()
  whole = _leaves(ret)
  wt, fixed, inputs = _criterion_call(whole, rb, args, epoch)
  assert wt.terms == (0x7FFF if K else 0x7FFF & ~(1 << cr.CYCLE)) or epoch != 0
  want = ag.mono_loss(wt, fixed, **inputs)
  want[0].backward()
  for size in sizes:
    spans = [(lo, min(R, lo + size)) for lo in range(0, R, size)]
    partial = torch.empty(int(ag.lib.dyn_mono_loss_workspace_bytes(R)), dtype=torch.uint8, device=DEV)
    parts = []
    for lo, hi in spans:
      part = _leaves({o: _cut(d, lo, hi) for o, d in ret.items()})
      wt_s, fixed_s, inputs_s = _criterion_call(part, _cut(rb, lo, hi), args, epoch)
      dims = ag.mono_loss_rows(wt_s, fixed_s, partial, lo, **inputs_s)
      parts.append((part, wt_s, fixed_s, inputs_s))
    table = ag.mono_loss_finish(partial, wt, R, *dims)
    assert torch.equal(table, want.detach()), (size, (table - want.detach()).abs().max().item())
    for part, wt_s, fixed_s, inputs_s in parts:
      ag.mono_loss(wt_s, dict(fixed_s, table=table), **inputs_s)[0].backward()
    for o, keys in TL.GRAD_KEYS.items():
      for k in keys:
        if whole[o][k].grad is None:  # an input of a term that is off
          assert all(p[0][o][k].grad is None for p in parts), (size, o, k)
          continue
        got = torch.cat([p[0][o][k].grad for p in parts], 1 if k in _AXIS1 else 0)
        assert torch.equal(got, whole[o][k].grad), (size, o, k)


def test_split_criterion_refuses_a_slice_off_the_block_grid():
  from dynibar_b200 import _lib
  ret, rb = TL.generated(64, 64, 3, 5)
  ret = {o: {k: v.to(DEV) for k, v in _cut(d, 4, 64).items()} for o, d in ret.items()}
  rb = {k: v.to(DEV) for k, v in _cut(rb, 4, 64).items()}
  wt, fixed, inputs = _criterion_call(ret, rb, TL.loss_args(), 0)
  partial = torch.empty(int(ag.lib.dyn_mono_loss_workspace_bytes(64)), dtype=torch.uint8, device=DEV)
  with pytest.raises(ValueError):
    ag.mono_loss_rows(wt, fixed, partial, 4, **inputs)
  out = torch.empty(40, device=DEV)
  with pytest.raises(RuntimeError):  # 7 rows for 64 rays: the finish wants cdiv(R, 8)
    _lib.check(ag.lib.dyn_mono_loss_finish(partial.data_ptr(), 7, ag.ctypes.byref(wt), 64, 64, 3, 6, out.data_ptr(),
                                           _lib.stream()))


# ---------------------------------------------------------------------------------------------------------------
# 2.-5. the sliced step
# ---------------------------------------------------------------------------------------------------------------
def _model(c, dev):
  import copy
  m = synthetic.model_to(copy.deepcopy(c["model"]), dev)
  for name in T.NETS:
    getattr(m, name).requires_grad_(True)
  m.trajectory_basis = m.trajectory_basis.detach().requires_grad_(True)
  return m


def step(c, prec, slice_rays, bootstrap=False):
  """train_step.mono_step_backward on case `c` -> result dict in train_step_ref's layout (terms and gradients)."""
  dev = torch.device(DEV)
  m = _model(c, dev)
  fm = tuple(f.to(dev).requires_grad_(True) for f in c["featmaps"])
  loss, terms = ts.mono_step_backward(c["frame"], c["t"], c["offs"], synthetic.to_device(dict(c["batch"], **c["sup"]),
                                                                                          dev),
                                      m, fm, Projector(dev), c["S"], c["args"], c["epoch"], slice_rays=slice_rays,
                                      bootstrap=bootstrap, inv_uniform=True, det=False, num_vv=c["num_vv"],
                                      jitter=c["jitter"].to(dev), precision=prec)
  h = lambda x: None if x is None else x.detach().cpu()
  res = {"terms": {k: h(v) for k, v in terms.items()}, "out": {}, "grad": {}}
  for name in T.NETS:
    for k, p in getattr(m, name).named_parameters():
      res["grad"]["%s.%s" % (name, k)] = h(p.grad)
  res["grad"]["trajectory_basis"] = h(m.trajectory_basis.grad)
  for i, f in enumerate(fm):
    res["grad"]["featmaps[%d]" % i] = h(f.grad)
  return res


def outputs(c, prec, spans):
  """The criterion inputs (OUT_KEYS) of the training forward run span by span under no_grad, concatenated."""
  dev = torch.device(DEV)
  m = _model(c, dev)
  fm = tuple(f.to(dev) for f in c["featmaps"])
  b = synthetic.to_device(dict(c["batch"], **c["sup"]), dev)
  jit = c["jitter"].to(dev)
  parts = []
  with torch.no_grad(), rr.precision_scope(prec):
    for lo, hi in spans:
      parts.append(rr._render_mono_train(c["frame"], c["t"], c["offs"], ts._slice_batch(b, lo, hi), m, fm, c["S"],
                                         c["args"], True, False, True, c["num_vv"], jit[lo:hi]))
  ret = T._cat(parts)
  return {"%s/%s" % (T._SHORT[o], k): ret[o][k].cpu() for o, ks in T.OUT_KEYS.items() for k in ks}


# per gradient (relative L2, max |error| / max |reference|): 2x the worst difference of a sliced step from the
# whole-batch step measured over test 2's and test 4's runs, rounded up to one digit, at least 1e-6; beside each the
# measured worst and the spread of two whole-batch runs.  A tensor not listed gets SPREAD_FLOOR.
SPREAD_BARS = {
    "grad.featmaps[1]": (1e-06, 1e-06),  # 2.14e-07 4.27e-07 (spread 2.09e-07 3.56e-07)
    "grad.featmaps[2]": (1e-06, 2e-06),  # 2.19e-07 5.18e-07 (spread 1.53e-07 3.48e-07)
    "grad.motion_mlp.coeff_linear.bias": (3e-06, 4e-06),  # 1.18e-06 1.56e-06 (spread 1.23e-06 1.87e-06)
    "grad.motion_mlp.coeff_linear.weight": (4e-06, 9e-06),  # 1.80e-06 4.19e-06 (spread 8.84e-07 2.65e-06)
    "grad.motion_mlp.pts_linears.0.bias": (1e-06, 2e-06),  # 3.03e-07 5.18e-07 (spread 3.23e-07 5.18e-07)
    "grad.motion_mlp.pts_linears.0.weight": (2e-06, 5e-06),  # 9.97e-07 2.38e-06 (spread 1.69e-07 4.32e-07)
    "grad.motion_mlp.pts_linears.1.bias": (1e-06, 1e-06),  # 3.15e-07 4.38e-07 (spread 3.29e-07 3.76e-07)
    "grad.motion_mlp.pts_linears.1.weight": (3e-06, 4e-06),  # 1.12e-06 1.69e-06 (spread 2.65e-07 3.73e-07)
    "grad.motion_mlp.pts_linears.2.bias": (1e-06, 2e-06),  # 4.06e-07 7.25e-07 (spread 4.58e-07 9.07e-07)
    "grad.motion_mlp.pts_linears.2.weight": (3e-06, 5e-06),  # 1.30e-06 2.46e-06 (spread 2.80e-07 5.36e-07)
    "grad.motion_mlp.pts_linears.3.bias": (1e-06, 2e-06),  # 4.10e-07 5.47e-07 (spread 4.33e-07 8.21e-07)
    "grad.motion_mlp.pts_linears.3.weight": (3e-06, 4e-06),  # 1.37e-06 1.76e-06 (spread 3.11e-07 5.60e-07)
    "grad.motion_mlp.pts_linears.4.bias": (1e-06, 2e-06),  # 3.68e-07 6.85e-07 (spread 3.88e-07 5.48e-07)
    "grad.motion_mlp.pts_linears.4.weight": (4e-06, 5e-06),  # 1.50e-06 2.18e-06 (spread 4.24e-07 6.00e-07)
    "grad.motion_mlp.pts_linears.5.bias": (1e-06, 2e-06),  # 3.72e-07 6.68e-07 (spread 3.42e-07 4.45e-07)
    "grad.motion_mlp.pts_linears.5.weight": (3e-06, 5e-06),  # 1.23e-06 2.36e-06 (spread 1.84e-07 6.31e-07)
    "grad.motion_mlp.pts_linears.6.bias": (1e-06, 2e-06),  # 4.35e-07 8.68e-07 (spread 4.75e-07 7.41e-07)
    "grad.motion_mlp.pts_linears.6.weight": (3e-06, 5e-06),  # 1.50e-06 2.24e-06 (spread 3.13e-07 7.64e-07)
    "grad.motion_mlp.pts_linears.7.bias": (2e-06, 2e-06),  # 6.55e-07 9.19e-07 (spread 8.02e-07 1.15e-06)
    "grad.motion_mlp.pts_linears.7.weight": (4e-06, 6e-06),  # 1.76e-06 2.57e-06 (spread 4.12e-07 9.15e-07)
    "grad.net_coarse_dy.base_fc.0.bias": (1e-06, 2e-06),  # 3.63e-07 5.32e-07 (spread 2.07e-07 3.47e-07)
    "grad.net_coarse_dy.base_fc.0.weight": (2e-05, 5e-05),  # 6.40e-06 2.03e-05 (spread 1.68e-07 3.72e-07)
    "grad.net_coarse_dy.base_fc.2.bias": (1e-06, 2e-06),  # 4.04e-07 7.02e-07 (spread 2.89e-07 4.54e-07)
    "grad.net_coarse_dy.base_fc.2.weight": (3e-05, 4e-05),  # 1.29e-05 1.86e-05 (spread 1.83e-07 4.01e-07)
    "grad.net_coarse_dy.geometry_fc.0.bias": (1e-06, 1e-06),  # 1.31e-07 3.24e-07 (spread 1.47e-07 3.25e-07)
    "grad.net_coarse_dy.geometry_fc.0.weight": (4e-06, 4e-06),  # 1.60e-06 1.89e-06 (spread 1.33e-07 3.56e-07)
    "grad.net_coarse_dy.geometry_fc.2.bias": (1e-06, 1e-06),  # 1.46e-07 2.38e-07 (spread 1.35e-07 2.95e-07)
    "grad.net_coarse_dy.geometry_fc.2.weight": (2e-06, 3e-06),  # 6.72e-07 1.33e-06 (spread 1.81e-07 3.50e-07)
    "grad.net_coarse_dy.out_geometry_fc.0.bias": (1e-06, 1e-06),  # 1.34e-07 3.31e-07 (spread 1.32e-07 3.49e-07)
    "grad.net_coarse_dy.out_geometry_fc.0.weight": (2e-06, 2e-06),  # 5.87e-07 8.78e-07 (spread 1.64e-07 5.02e-07)
    "grad.net_coarse_dy.out_geometry_fc.2.bias": (1e-06, 1e-06),  # 1.74e-07 1.74e-07 (spread 1.59e-07 1.59e-07)
    "grad.net_coarse_dy.out_geometry_fc.2.weight": (2e-06, 2e-06),  # 6.09e-07 9.42e-07 (spread 2.12e-07 2.90e-07)
    "grad.net_coarse_dy.ray_attention.fc.weight": (2e-06, 2e-06),  # 5.52e-07 8.01e-07 (spread 1.62e-07 2.85e-07)
    "grad.net_coarse_dy.ray_attention.layer_norm.bias": (2e-06, 3e-06),  # 6.93e-07 1.37e-06 (spread 5.54e-07 1.20e-06)
    "grad.net_coarse_dy.ray_attention.layer_norm.weight": (2e-06, 4e-06),  # 7.57e-07 1.50e-06 (spread 4.71e-07 6.15e-07)
    "grad.net_coarse_dy.ray_attention.w_ks.weight": (2e-06, 3e-06),  # 8.68e-07 1.24e-06 (spread 1.85e-07 2.81e-07)
    "grad.net_coarse_dy.ray_attention.w_qs.weight": (2e-06, 2e-06),  # 5.69e-07 8.47e-07 (spread 1.75e-07 5.10e-07)
    "grad.net_coarse_dy.ray_attention.w_vs.weight": (2e-06, 3e-06),  # 5.42e-07 1.38e-06 (spread 1.80e-07 5.03e-07)
    "grad.net_coarse_dy.ray_dir_fc.0.bias": (1e-06, 1e-06),  # 3.49e-07 3.29e-07 (spread 3.74e-07 4.34e-07)
    "grad.net_coarse_dy.ray_dir_fc.0.weight": (1e-06, 1e-06),  # 3.12e-07 3.67e-07 (spread 3.50e-07 3.67e-07)
    "grad.net_coarse_dy.ray_dir_fc.2.bias": (1e-06, 1e-06),  # 3.27e-07 4.98e-07 (spread 3.53e-07 5.36e-07)
    "grad.net_coarse_dy.ray_dir_fc.2.weight": (1e-06, 1e-06),  # 2.78e-07 4.79e-07 (spread 3.37e-07 5.85e-07)
    "grad.net_coarse_dy.ref_pts_fc.0.bias": (1e-06, 1e-06),  # 1.35e-07 3.03e-07 (spread 1.39e-07 3.03e-07)
    "grad.net_coarse_dy.ref_pts_fc.0.weight": (2e-06, 3e-06),  # 6.82e-07 1.06e-06 (spread 1.63e-07 2.39e-07)
    "grad.net_coarse_dy.ref_pts_fc.2.bias": (1e-06, 1e-06),  # 1.42e-07 2.69e-07 (spread 1.13e-07 2.24e-07)
    "grad.net_coarse_dy.ref_pts_fc.2.weight": (2e-06, 2e-06),  # 6.73e-07 6.69e-07 (spread 1.75e-07 2.87e-07)
    "grad.net_coarse_dy.rgb_fc.0.bias": (1e-06, 1e-06),  # 1.11e-07 2.59e-07 (spread 1.08e-07 1.88e-07)
    "grad.net_coarse_dy.rgb_fc.0.weight": (1e-06, 3e-06),  # 4.41e-07 1.06e-06 (spread 8.75e-08 1.45e-07)
    "grad.net_coarse_dy.rgb_fc.2.bias": (1e-06, 1e-06),  # 1.11e-07 1.94e-07 (spread 1.26e-07 2.41e-07)
    "grad.net_coarse_dy.rgb_fc.2.weight": (2e-06, 3e-06),  # 7.18e-07 1.48e-06 (spread 1.22e-07 2.09e-07)
    "grad.net_coarse_dy.rgb_fc.4.bias": (1e-06, 1e-06),  # 1.28e-07 1.11e-07 (spread 8.80e-08 9.13e-08)
    "grad.net_coarse_dy.rgb_fc.4.weight": (2e-06, 2e-06),  # 5.38e-07 5.42e-07 (spread 1.51e-07 3.77e-07)
    "grad.net_coarse_dy.vis_fc.0.bias": (1e-06, 2e-06),  # 4.21e-07 8.29e-07 (spread 3.34e-07 7.74e-07)
    "grad.net_coarse_dy.vis_fc.0.weight": (2e-05, 2e-05),  # 6.14e-06 7.74e-06 (spread 2.35e-07 5.95e-07)
    "grad.net_coarse_dy.vis_fc.2.bias": (1e-06, 2e-06),  # 4.53e-07 8.78e-07 (spread 2.50e-07 4.44e-07)
    "grad.net_coarse_dy.vis_fc.2.weight": (4e-05, 4e-05),  # 1.64e-05 1.90e-05 (spread 1.88e-07 5.31e-07)
    "grad.net_coarse_dy.vis_fc2.0.bias": (9e-06, 9e-06),  # 4.36e-06 4.39e-06 (spread 3.00e-07 3.72e-07)
    "grad.net_coarse_dy.vis_fc2.0.weight": (7e-06, 8e-06),  # 3.38e-06 3.85e-06 (spread 2.63e-07 6.57e-07)
    "grad.net_coarse_dy.vis_fc2.2.bias": (1e-06, 2e-06),  # 2.02e-07 6.97e-07 (spread 1.02e-08 5.03e-08)
    "grad.net_coarse_dy.vis_fc2.2.weight": (7e-06, 8e-06),  # 3.23e-06 3.57e-06 (spread 2.58e-07 5.10e-07)
    "grad.net_coarse_st.base_fc.0.bias": (1e-06, 2e-06),  # 3.93e-07 8.74e-07 (spread 1.55e-07 3.50e-07)
    "grad.net_coarse_st.base_fc.0.weight": (2e-05, 4e-05),  # 6.42e-06 1.87e-05 (spread 1.10e-07 4.24e-07)
    "grad.net_coarse_st.base_fc.2.bias": (2e-06, 2e-06),  # 5.64e-07 7.82e-07 (spread 2.89e-07 5.50e-07)
    "grad.net_coarse_st.base_fc.2.weight": (3e-05, 4e-05),  # 1.44e-05 1.84e-05 (spread 1.82e-07 5.18e-07)
    "grad.net_coarse_st.geometry_fc.0.bias": (1e-06, 1e-06),  # 1.38e-07 2.56e-07 (spread 1.08e-07 1.99e-07)
    "grad.net_coarse_st.geometry_fc.0.weight": (3e-06, 3e-06),  # 1.30e-06 1.28e-06 (spread 1.03e-07 2.01e-07)
    "grad.net_coarse_st.geometry_fc.2.bias": (1e-06, 1e-06),  # 1.78e-07 3.47e-07 (spread 1.11e-07 2.02e-07)
    "grad.net_coarse_st.geometry_fc.2.weight": (2e-06, 3e-06),  # 5.97e-07 1.48e-06 (spread 1.39e-07 2.91e-07)
    "grad.net_coarse_st.out_geometry_fc.0.bias": (1e-06, 1e-06),  # 1.38e-07 2.97e-07 (spread 9.79e-08 3.03e-07)
    "grad.net_coarse_st.out_geometry_fc.0.weight": (2e-06, 3e-06),  # 5.29e-07 1.17e-06 (spread 1.23e-07 2.47e-07)
    "grad.net_coarse_st.out_geometry_fc.2.bias": (1e-06, 1e-06),  # 3.11e-07 3.11e-07 (spread 1.44e-07 1.44e-07)
    "grad.net_coarse_st.out_geometry_fc.2.weight": (2e-06, 2e-06),  # 5.76e-07 9.64e-07 (spread 1.55e-07 2.32e-07)
    "grad.net_coarse_st.ray_attention.fc.weight": (2e-06, 3e-06),  # 5.38e-07 1.14e-06 (spread 1.32e-07 3.24e-07)
    "grad.net_coarse_st.ray_attention.layer_norm.bias": (2e-06, 3e-06),  # 6.18e-07 1.48e-06 (spread 4.51e-07 7.26e-07)
    "grad.net_coarse_st.ray_attention.layer_norm.weight": (2e-06, 3e-06),  # 6.03e-07 1.11e-06 (spread 4.43e-07 6.35e-07)
    "grad.net_coarse_st.ray_attention.w_ks.weight": (2e-06, 3e-06),  # 6.38e-07 1.04e-06 (spread 1.47e-07 2.41e-07)
    "grad.net_coarse_st.ray_attention.w_qs.weight": (1e-06, 1e-06),  # 4.80e-07 4.77e-07 (spread 1.35e-07 2.20e-07)
    "grad.net_coarse_st.ray_attention.w_vs.weight": (2e-06, 3e-06),  # 5.20e-07 1.18e-06 (spread 1.43e-07 3.44e-07)
    "grad.net_coarse_st.ray_dir_fc.0.bias": (1e-06, 2e-06),  # 4.40e-07 8.10e-07 (spread 1.74e-07 3.56e-07)
    "grad.net_coarse_st.ray_dir_fc.0.weight": (3e-05, 2e-05),  # 1.34e-05 6.88e-06 (spread 1.59e-07 2.19e-07)
    "grad.net_coarse_st.ray_dir_fc.2.bias": (2e-06, 2e-06),  # 5.39e-07 7.58e-07 (spread 4.49e-07 6.82e-07)
    "grad.net_coarse_st.ray_dir_fc.2.weight": (4e-05, 4e-05),  # 1.61e-05 1.70e-05 (spread 1.78e-07 3.18e-07)
    "grad.net_coarse_st.ref_feature_fc.0.bias": (1e-06, 1e-06),  # 1.36e-07 2.08e-07 (spread 0.00e+00 0.00e+00)
    "grad.net_coarse_st.ref_feature_fc.0.weight": (2e-06, 3e-06),  # 5.69e-07 1.23e-06 (spread 0.00e+00 0.00e+00)
    "grad.net_coarse_st.rgb_fc.0.bias": (1e-06, 1e-06),  # 9.71e-08 4.14e-07 (spread 1.72e-08 7.90e-08)
    "grad.net_coarse_st.rgb_fc.0.weight": (2e-05, 2e-05),  # 5.36e-06 7.59e-06 (spread 2.69e-07 4.29e-07)
    "grad.net_coarse_st.rgb_fc.2.bias": (1e-06, 4e-06),  # 2.52e-07 1.80e-06 (spread 2.05e-08 2.84e-07)
    "grad.net_coarse_st.rgb_fc.2.weight": (8e-06, 2e-05),  # 3.81e-06 5.23e-06 (spread 2.57e-07 5.23e-07)
    "grad.net_coarse_st.rgb_fc.4.bias": (2e-06, 5e-06),  # 5.51e-07 2.01e-06 (spread 4.36e-08 1.34e-07)
    "grad.net_coarse_st.rgb_fc.4.weight": (9e-06, 2e-05),  # 4.45e-06 5.41e-06 (spread 2.61e-07 4.12e-07)
    "grad.net_coarse_st.s": (1e-06, 1e-06),  # 3.01e-07 3.01e-07 (spread 2.41e-07 2.41e-07)
    "grad.net_coarse_st.vis_fc.0.bias": (1e-06, 2e-06),  # 4.44e-07 5.79e-07 (spread 3.38e-07 6.42e-07)
    "grad.net_coarse_st.vis_fc.0.weight": (2e-05, 2e-05),  # 7.13e-06 8.36e-06 (spread 2.14e-07 4.32e-07)
    "grad.net_coarse_st.vis_fc.2.bias": (1e-06, 2e-06),  # 4.41e-07 7.10e-07 (spread 2.08e-07 4.26e-07)
    "grad.net_coarse_st.vis_fc.2.weight": (4e-05, 4e-05),  # 1.80e-05 1.89e-05 (spread 1.64e-07 4.89e-07)
    "grad.net_coarse_st.vis_fc2.0.bias": (1e-05, 8e-06),  # 4.87e-06 3.83e-06 (spread 3.14e-07 4.77e-07)
    "grad.net_coarse_st.vis_fc2.0.weight": (2e-05, 2e-05),  # 5.26e-06 5.94e-06 (spread 2.24e-07 4.88e-07)
    "grad.net_coarse_st.vis_fc2.2.bias": (3e-06, 8e-06),  # 1.05e-06 3.73e-06 (spread 1.61e-08 5.48e-08)
    "grad.net_coarse_st.vis_fc2.2.weight": (2e-05, 2e-05),  # 5.15e-06 5.46e-06 (spread 2.93e-07 3.13e-07)
    "grad.trajectory_basis": (2e-06, 2e-06),  # 5.80e-07 8.16e-07 (spread 0.00e+00 0.00e+00)
}
SPREAD_FLOOR = (1e-5, 1e-5)


def spread_bar(name):
  return SPREAD_BARS.get(name, SPREAD_FLOOR)


def _grad_errors(got, ref, V_st):
  return {k: v for k, v in T.errors(got, ref, V_st).items() if k.startswith("grad.")}


def _worst(errs):
  r = {k: max(a / spread_bar(k)[0], b / spread_bar(k)[1]) for k, (a, b) in errs.items()}
  return r, max(r.items(), key=lambda kv: kv[1]) if r else ("-", 0.0)


SLICED = [("shipped", "bf16", 512), ("shipped", "bf16", 384), ("shipped", "fp32", 512), ("late", "bf16", 512),
          ("late", "fp32", 384), ("edges_occ1", "bf16", 64), ("edges_occ1", "fp32", 64)]


@pytest.mark.parametrize("case,prec,slice_rays", SLICED)
def test_sliced_step_matches_the_whole_batch(case, prec, slice_rays):
  c = T.make_case(case)
  R = c["batch"]["ray_o"].shape[0]
  spans = ts.slice_plan(R, slice_rays, c["S"])
  assert len(spans) > 1
  whole = [step(c, prec, R) for _ in range(2)]
  sliced = step(c, prec, slice_rays)
  for k, v in whole[0]["terms"].items():
    assert torch.equal(sliced["terms"][k], v), (k, sliced["terms"][k].item(), v.item())
  a, b = outputs(c, prec, [(0, R)]), outputs(c, prec, spans)
  for k in a:
    assert torch.equal(a[k], b[k]), (k, (a[k] - b[k]).abs().max().item())
  spread = _grad_errors(whole[1], whole[0], c["V_st"])
  errs = _grad_errors(sliced, whole[0], c["V_st"])
  for k in sorted(errs):
    print("  SPREAD %s %s %d %s %.3e %.3e | sliced %.3e %.3e" % (case, prec, slice_rays, k, *spread[k], *errs[k]))
  r, worst = _worst(errs)
  print("\nsliced %s %s %d (%d slices): worst %s, %.2f of its bar" % (case, prec, slice_rays, len(spans), *worst))
  bad = {k: (errs[k], spread_bar(k)) for k, v in r.items() if not v <= 1.0}
  assert not bad, bad


@pytest.mark.parametrize("case,prec", [("shipped", "bf16"), ("edges_occ1", "fp32")])
def test_sliced_bootstrap_matches_the_whole_batch(case, prec):
  c = T.make_case(case)
  R = c["batch"]["ray_o"].shape[0]
  slice_rays = 512 if R > 512 else 64
  whole = step(c, prec, R, bootstrap=True)
  sliced = step(c, prec, slice_rays, bootstrap=True)
  assert torch.equal(sliced["terms"]["loss"], whole["terms"]["loss"])
  errs = _grad_errors(sliced, whole, c["V_st"])
  assert errs and any(k.startswith("grad.net_coarse_st") for k in errs)
  for k in sorted(errs):
    print("  BOOT %s %s %s %.3e %.3e" % (case, prec, k, *errs[k]))
  r, worst = _worst(errs)
  print("\nbootstrap %s %s: worst %s, %.2f of its bar" % (case, prec, *worst))
  bad = {k: (errs[k], spread_bar(k)) for k, v in r.items() if not v <= 1.0}
  assert not bad, bad


def test_per_slice_denominators_miss_the_bars(monkeypatch):
  c = T.make_case("shipped")
  whole = step(c, "bf16", 1024)
  own = lambda ret, rb, args, epoch, table, bootstrap=False: cr.mono_step_loss(ret, rb, args, epoch)[0]
  monkeypatch.setattr(cr, "slice_loss", own)
  planted = step(c, "bf16", 512)
  r, worst = _worst(_grad_errors(planted, whole, c["V_st"]))
  print("\nplant per-slice denominators: %s moves %.1fx its bar" % worst)
  assert worst[1] >= T.PLANT_MARGIN, worst


# ---------------------------------------------------------------------------------------------------------------
# 3. the shipped batch against the float64 reference
# ---------------------------------------------------------------------------------------------------------------
SHIPPED_3072 = dict(T.CASES["shipped"], rays=3072, seed=31)


def shipped_bar(name):
  """SHIPPED_BARS: the bf16 bars of the whole-batch step (measured worst 0.49 of them, grad.featmaps[1])."""
  import test_train_step_gpu as TS
  return TS.BARS["bf16"][name]


def test_shipped_batch_matches_the_float64_reference(monkeypatch):
  monkeypatch.setitem(T.CASES, "shipped_3072", SHIPPED_3072)
  # the library runs 1024-ray slices; the reference's 128-ray chunks must see the products a 1024-ray slice runs
  check_chunk = T._check_chunk
  monkeypatch.setattr(T, "_check_chunk", lambda R, chunk, S: check_chunk(1024, chunk, S))
  c = T.make_case("shipped_3072")
  assert c["batch"]["ray_o"].shape[0] == 3072
  torch.cuda.synchronize()
  torch.cuda.empty_cache()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.perf_counter()
  got = step(c, "bf16", 1024)
  torch.cuda.synchronize()
  stats = {"library_s": time.perf_counter() - t0, "library_peak_GB": torch.cuda.max_memory_allocated() / 2 ** 30}
  torch.cuda.empty_cache()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.perf_counter()
  ref = T.reference(c, DEV, "kernel", chunk=128)
  torch.cuda.synchronize()
  stats.update(reference_s=time.perf_counter() - t0, reference_peak_GB=torch.cuda.max_memory_allocated() / 2 ** 30)
  ref["out"] = {}
  errs = T.errors(got, ref, c["V_st"])
  r = {k: max(a / shipped_bar(k)[0], b / shipped_bar(k)[1]) for k, (a, b) in errs.items()}
  worst = max(r.items(), key=lambda kv: kv[1])
  print("\nshipped 3072 bf16 in 1024-ray slices: worst %s, %.2f of its bar; %s"
        % (worst[0], worst[1], ", ".join("%s %.2f" % kv for kv in stats.items())))
  for name, (rel, mx) in sorted(errs.items()):
    print("  ERR3072 %s %.3e %.3e" % (name, rel, mx))
  bad = {k: (errs[k], shipped_bar(k)) for k, v in r.items() if not v <= 1.0}
  assert not bad, bad
