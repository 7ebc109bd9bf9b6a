"""Training gives the same bits twice.  Every training entry point runs the same call more than once and every output,
gradient and (for whole steps) Adam moment must be equal bit for bit (torch.equal on the bits, NaN payloads included).

Between the runs the device is made to look different, so that agreement from identical scheduling cannot pass:
  - run 1: the grow-only workspace (_lib.workspace) filled with 0x00, after a large unrelated GEMM;
  - run 2: under memory_contract.poisoned(0x7F): fresh exact-size workspaces and torch.empty buffers full of 3.39e38,
    after the grow-only workspace was filled with 0xFF (NaN) and other kernels ran;
  - run 3: after a larger call of the same entry point (where the product's slabs depend on the row count) and every
    grow-only buffer regrown to a larger size and filled with 0x5A: the same rows placed in a larger call's workspace.

The training backward adds every reduction over rows in a fixed order (include/dynibar_b200.h, "Conventions"): slab
partials of the split-K and tensor-core weight gradients, column sums, LayerNorm / InstanceNorm parameter gradients and
the anti-aliasing `s` are added in slab order, col2im is a gather, and the feature-map gradient of the projection is a
radix sort by texel plus a gather.  With float atomics in any of them, two runs differ in the last bits; a read of
memory a call did not write differs between the fill patterns.

Shapes are the float64 reference tests' own: train_stage_ref.NET_CASES and MOTION_CASES, test_staged_nets_gpu's
17-32-view and long-ray TRAIN_CASES, encoder_ref.CASES, the shipped and edge monocular steps, the multi-view fine
stage of test_train_mv_gpu, and Trainer steps across the warm-up / main boundary.  An adversarial projection rig puts
every sample of one view on a handful of texels (the most same-address contention the feature-map gradient can see).
"""

import copy

import numpy as np
import pytest
import torch

import encoder_ref as er
import memory_contract as mc
import train_stage_ref as tsr
from dynibar_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _garble(byte):
  """Fill every buffer of the grow-only workspace with `byte`, then run unrelated kernels."""
  for buf in _lib.workspace._bufs.values():
    if buf is not None:
      buf.fill_(byte)
  a = torch.randn(3000, 3000, device=DEV)
  (a @ a).relu_().sum().item()


def _regrow(byte):
  """Replace every grow-only buffer by a larger one filled with `byte`.  Only the sizes are kept across the loop, so
  each old buffer is released before its successor is allocated."""
  sizes = {key: buf.numel() for key, buf in _lib.workspace._bufs.items() if buf is not None}
  torch.cuda.empty_cache()
  for (dev, slot), n in sizes.items():
    _lib.workspace.get(n + (3 << 20), dev, slot=slot).fill_(byte)


def check_repeatable(run, what, bigger=None):
  """run() -> nested outputs / gradients; bigger: a larger call of the same entry point, run before the third run."""
  runs = {}
  _garble(0x00)
  runs["first"] = mc.flatten(run())
  _garble(0xFF)
  with mc.poisoned(0x7F):
    runs["poisoned 0x7F"] = mc.flatten(run())
  if bigger is not None:
    bigger()
  _regrow(0x5A)
  _garble(0x5A)
  runs["after a larger call, regrown"] = mc.flatten(run())
  mc.assert_bit_identical(runs, what)
  print("\n%s: %d tensors, %d elements bit-identical over %d runs" % (
      what, len(runs["first"]), sum(v.numel() for v in runs["first"].values()), len(runs)))


# ---------------------------------------------------------------------------------------------------------------
# the aggregation nets and the MotionMLP (autograd wrappers of dyn_net_*_backward / dyn_motion_mlp_backward)
# ---------------------------------------------------------------------------------------------------------------
def _staged_train_cases():
  from test_staged_nets_gpu import TRAIN_CASES
  return {k: TRAIN_CASES[k] for k in ("v17", "v32", "s192", "s384")}


NET_CASES = dict(tsr.NET_CASES, **{"staged_" + k: v for k, v in _staged_train_cases().items()})


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("case", list(NET_CASES))
@pytest.mark.parametrize("kind", ["dynamic", "static"])
def test_net_backward_is_repeatable(kind, case, prec):
  from test_train_stage_gpu import _library
  R, S, V, aa, mrgb = NET_CASES[case]
  c = tsr.make_net_case(kind, R, S, V, aa, mrgb, seed=R + S + V)
  big = tsr.make_net_case(kind, 2 * R + 3, S, V, aa, mrgb, seed=R + S + V + 1) if R * S * V <= 300000 else None
  check_repeatable(lambda: _library(c, prec), "%s %s %s" % (kind, case, prec),
                   bigger=(lambda: _library(big, prec)) if big is not None else None)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("case", list(tsr.MOTION_CASES))
def test_motion_backward_is_repeatable(case, prec):
  """n65573: the fp32 weight gradients run split-K (17 splits), the bf16 ones several tensor-core slabs per tile."""
  from test_train_stage_gpu import _library
  N, nb = tsr.MOTION_CASES[case]
  c = tsr.make_motion_case(N, nb, seed=N + nb)
  big = tsr.make_motion_case(2 * N + 1, nb, seed=N + nb + 1)
  check_repeatable(lambda: _library(c, prec), "motion %s %s" % (case, prec), bigger=lambda: _library(big, prec))


# ---------------------------------------------------------------------------------------------------------------
# the 2-D encoder
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("case", list(er.CASES))
def test_encoder_backward_is_repeatable(case, prec):
  from test_encoder_train_gpu import _library
  c = er.make_case(case)
  check_repeatable(lambda: _library(c, prec), "encoder %s %s" % (case, prec),
                   bigger=lambda: _library(er.make_case("ragged", seed=5), prec))


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_encoder_three_calls_in_one_graph_are_repeatable(prec):
  """bench.py's train_step shape of use: three encoder calls (2, 3 and 1 images) backpropagated in one graph."""
  from dynibar_b200 import feature_network as fn, render_ray as rr
  mod = er.make_model(7).to(DEV).requires_grad_(True)
  g = torch.Generator().manual_seed(8)
  imgs = [torch.rand(n, 3, 128, 192, generator=g).to(DEV) for n in (2, 3, 1)]
  gcs = [torch.randn(n, 32, 32, 48, generator=g).to(DEV) for n in (2, 3, 1)]
  params = dict(mod.named_parameters())

  def run():
    with rr.precision_scope(prec):
      mod.zero_grad(set_to_none=True)
      sum((mod(im)[0] * gc).sum() for im, gc in zip(imgs, gcs)).backward()
    return {k: params[k].grad.clone() for k in fn._EXECUTED}
  check_repeatable(run, "encoder, three calls in one graph, %s" % prec)


# ---------------------------------------------------------------------------------------------------------------
# the projection / bilinear gather: feature-map gradient under maximal same-texel contention
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tile", [1, 16])
def test_gather_backward_is_repeatable_when_samples_pile_onto_few_texels(golden, tile):
  """The mv_linear rig with its rays tiled `tile` times; in view 0 every sample sits within 1e-4 of one point, so all
  R S of its taps land on at most four texels of the feature map.  The other views keep their own points."""
  from dynibar_b200 import autograd as ag, synthetic
  import scenes
  fx = golden("mv_linear")
  batch, feat_c, _, _, _, _, _, _ = scenes.build(fx["cfg"])
  pts, seq = fx["stages"]["pts"], fx["stages"]["seq"]
  pts = pts.repeat(tile, 1, 1)
  seq = seq.repeat(1, tile, 1, 1).clone()
  g = torch.Generator().manual_seed(tile)
  seq[0] = seq[0, :1, :1] + 1e-4 * torch.randn(seq[0].shape, generator=g)
  d = lambda x: synthetic.to_device(x, DEV)
  fm = feat_c[0]
  gen = None

  def run():
    nonlocal gen
    fd, sd = fm.to(DEV).requires_grad_(True), seq.to(DEV).requires_grad_(True)
    f, _, _ = ag.project_gather(d(pts), sd, d(batch["camera"]), d(batch["src_rgbs"]), d(batch["src_cameras"]), fd)
    if gen is None:
      gen = torch.randn(f.shape, generator=g).to(DEV)
    (f * gen).sum().backward()
    return {"featmaps": fd.grad, "xyz": sd.grad}
  out = run()
  assert out["featmaps"][0].abs().sum() > 0
  check_repeatable(run, "gather backward, %d x rays, view 0 on one point" % tile)


# ---------------------------------------------------------------------------------------------------------------
# the `s` of the anti-aliased pooling at many (point, view) rows
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_anti_alias_s_gradient_is_repeatable(prec):
  """The static net's `s` (nonzero) summed over 1024 x 32 points and 9 views: 128 blocks' shares."""
  from test_train_stage_gpu import _library
  c = tsr.make_net_case("static", 1024, 32, 9, True, False, seed=99)
  with torch.no_grad():
    c["mod"].s.fill_(0.7)

  def run():
    got = _library(c, prec)
    assert got["s"].abs().item() > 0
    return {"s": got["s"], "out": got["out"]}
  check_repeatable(run, "static s %s" % prec)


# ---------------------------------------------------------------------------------------------------------------
# whole steps
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case,prec,slice_rays", [("shipped", "bf16", 256), ("shipped", "bf16", 1024),
                                                  ("shipped", "fp32", 1024), ("edges_occ1", "fp32", 64)])
def test_mono_step_is_repeatable(case, prec, slice_rays):
  import train_step_ref as T
  from test_train_sliced_gpu import step
  c = T.make_case(case)

  def run():
    res = step(c, prec, slice_rays)
    return res["terms"], res["grad"]
  check_repeatable(run, "mono_step_backward %s %s, slices of %d" % (case, prec, slice_rays))


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_mv_fine_stage_step_is_repeatable(prec):
  from dynibar_b200 import render_ray as rr
  from dynibar_b200.projection import Projector
  from test_train_mv_gpu import _FINE, _mv_device, _mv_scene
  cfg, batch, feat_c, feat_f, frame, t, offs, model, args = _mv_scene("mv_nvidia", 37)
  g = torch.Generator()

  def run():
    m, b, fc, ff = _mv_device(copy.deepcopy(model), batch, feat_c, feat_f)
    got = rr.render_rays_mv(frame, t, offs, b, m, Projector(DEV), fc, ff, cfg["N_samples"], args, precision=prec,
                            inv_uniform=cfg["inv_uniform"], N_importance=cfg["N_importance"], det=True,
                            is_train=True)
    out = got["outputs_fine_ref"]
    g.manual_seed(7)
    sum((v * torch.randn(v.shape, generator=g).to(DEV)).sum() for k, v in sorted(out.items())
        if torch.is_tensor(v) and v.requires_grad).backward()
    grads = {"%s.%s" % (n, k): p.grad for n in _FINE for k, p in getattr(m, n).named_parameters()}
    grads["trajectory_basis_fine"] = m.trajectory_basis_fine.grad
    grads.update({"feat_f[%d]" % i: f.grad for i, f in enumerate(ff) if f is not None})
    return got, grads
  check_repeatable(run, "render_rays_mv fine stage %s" % prec)


def test_trainer_steps_across_the_warmup_boundary_are_repeatable(tmp_path):
  """Trainer.run over the last warm-up step and the first two main steps (bf16, 512 rays in 256-ray slices): every
  parameter, its .grad and both Adam moments."""
  import mono_scene_ref as msr
  from dynibar_b200 import mono_scene
  from test_train_loop_gpu import N, H, W, _args, _fresh
  args = _args(init_decay_epoch=2)
  path = msr.write_scene(str(tmp_path / "s" / "dense"), msr.synthetic_scene(21, N, H, W, mask_hw=(40, 70)))
  scene = mono_scene.MonocularScene(path, args, torch.device(DEV))

  def run():
    t = _fresh(scene, args)
    t.run(N + 2)
    assert [r["bootstrap"] for r in t.record][N - 1:] == [True, False, False]
    out = {}
    for k, group in enumerate(t.optimizer.param_groups):
      for i, p in enumerate(group["params"]):
        st = t.optimizer.state.get(p, {})
        out["g%d.%d" % (k, i)] = (p.detach(), p.grad, st.get("exp_avg"), st.get("exp_avg_sq"))
    return out
  check_repeatable(run, "Trainer, %d steps across the warm-up boundary" % (N + 2))
