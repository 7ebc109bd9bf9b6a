"""Host logic of the trainable trajectory basis and of render_rays_mv's training path that needs no GPU: the
basis-difference rows, routing of render_rays_mv to its differentiable fine stage, the multi-camera refusal and the
slicing of large ray batches (dynibar_b200.render_ray._render_mv_train_chunked)."""

from collections import OrderedDict

import pytest
import torch

from dynibar_b200 import render_ray as rr, sample_ray as sr, synthetic


def test_basis_rows_match_the_reference_rows_and_carry_the_gradient():
  basis = synthetic.init_dct_basis(6, 24)
  pairs = [(1 + o, 1) for o in (-3, -2, -1, 0, 1, 2, 3)] + [(-2, 5), (23, -24)] + [(None, None)] * 2
  want = torch.stack([basis[a] - basis[b] if a is not None else torch.zeros(6) for a, b in pairs])
  frozen = rr._basis_rows(basis, pairs, "cpu")
  assert not frozen.requires_grad and torch.equal(frozen, want)
  live = basis.clone().requires_grad_(True)
  D = rr._basis_rows(live, pairs, "cpu")
  assert D.requires_grad and torch.equal(D.detach(), want)
  assert torch.equal(D[-2:].detach(), torch.zeros(2, 6))
  g = torch.randn(D.shape, generator=torch.Generator().manual_seed(0))
  (D * g).sum().backward()
  want = torch.zeros_like(basis)
  for i, (a, b) in enumerate(pairs):
    if a is not None:  # negative rows wrap as in the reference's basis[f - 3]
      want[a] += g[i]
      want[b] -= g[i]
  torch.testing.assert_close(live.grad, want, rtol=0, atol=1e-6)
  with pytest.raises(IndexError):
    rr._basis_rows(live, [(24, 0)], "cpu")


@pytest.mark.parametrize("S", [1, 2, 3, 4, 5, 6, 15, 25, 35, 45])
def test_keep_mask_zeroes_the_reference_tail(S):
  """The training paths' zeroed tail is the reference's `[:, -n:]` with n = int(round(0.1 S)): all S samples when n is
  0 (S <= 5, `-0:` is the whole axis), and Python's round-half-even at S = 25 (2) and 35 (4)."""
  import motion_stage_ref
  keep = rr._keep_mask(S, "cpu")
  n = motion_stage_ref.n_last(S)
  want = torch.ones(1, S, 1)
  want[:, S - n:] = 0.0
  assert torch.equal(keep, want), (S, keep.flatten().tolist())
  ref = torch.ones(1, S, 1)
  ref[:, -int(round(S * 0.1)):] *= 0.0  # the reference's own slice, ibrnet/render_ray.py:459, :472
  assert torch.equal(keep, ref)


def _mv_model():
  model, args = synthetic.make_model(8, 8, num_frames=24)
  return model, args


def test_fine_stage_routing():
  model, _ = _mv_model()
  fm = (torch.zeros(1), None, torch.zeros(1))
  assert not rr._fine_stage_wants_grad(model, fm)
  model.net_coarse_dy.requires_grad_(True)  # the coarse stage never trains in render_rays_mv
  assert not rr._fine_stage_wants_grad(model, fm)
  model.trajectory_basis.requires_grad_(True)
  assert not rr._fine_stage_wants_grad(model, fm)
  for name in rr._FINE_MODULES:
    getattr(model, name).requires_grad_(True)
    assert rr._fine_stage_wants_grad(model, fm)
    with torch.no_grad():
      assert not rr._fine_stage_wants_grad(model, fm)
    getattr(model, name).requires_grad_(False)
  model.trajectory_basis_fine.requires_grad_(True)
  assert rr._fine_stage_wants_grad(model, fm)
  model.trajectory_basis_fine.requires_grad_(False)
  assert rr._fine_stage_wants_grad(model, (torch.zeros(1, requires_grad=True), None, torch.zeros(1)))
  assert rr._fine_stage_wants_grad(model, (torch.zeros(1), None, torch.zeros(1, requires_grad=True)))
  # a trainable basis also routes render_rays_mono to its training path
  mono = synthetic.make_model(8, 0, mono=True)[0]
  assert not rr._wants_grad(mono, fm)
  mono.trajectory_basis.requires_grad_(True)
  assert rr._wants_grad(mono, fm)


def test_multi_camera_batches_refuse_fine_stage_training():
  model, args = _mv_model()
  batch, feat_c, feat_f, frame, t, offs = synthetic.make_scene(H=12, W=16, V_dy=3, V_st=2, rays=6)
  multi = sr.stack_ray_batches([batch, dict(batch, camera=batch["camera"].clone())])[0]
  model.net_fine_st.requires_grad_(True)
  with pytest.raises(NotImplementedError, match="one target camera"):
    rr.render_rays_mv(frame, t, offs, multi, model, None, feat_c, feat_f, 8, args, N_importance=8, det=True)


def _fake_mv_train(frame_idx, time_embedding, time_offset, ray_batch, model, coarse_featmaps, fine_featmaps, N_samples,
                   args, inv_uniform, N_importance, det, jitter, u):
  """Stands in for the CUDA path: every output is a per-ray function of ray_o (and of the random draws), in the
  reference's layouts."""
  o = ray_batch["ray_o"]
  R = o.shape[0]
  s = o.sum(-1)
  S = N_samples + N_importance
  coarse = OrderedDict(rgb=o * 2, weights=s[:, None].expand(R, N_samples) * 1.0, mask=s > 0,
                       z_vals=jitter * 1.0 if jitter is not None else s[:, None].expand(R, N_samples) * 1.0)
  fine = OrderedDict(rgb=o * 3, depth=s, weights=s[:, None].expand(R, S) + u.sum(1, keepdim=True),
                     render_flows=torch.stack([o[:, :2] + k for k in range(3)]), exp_sf=o + 1)
  return {"outputs_coarse": None, "outputs_fine": None, "outputs_coarse_ref": coarse, "outputs_fine_ref": fine,
          "outputs_fine_ref_dy": OrderedDict(rgb=o - 1), "outputs_fine_anchor": None, "outputs_fine_anchor_dy": None}


def test_mv_ray_slices_are_merged_along_the_ray_axis(monkeypatch):
  monkeypatch.setattr(rr, "_render_mv_train", _fake_mv_train)
  g = torch.Generator().manual_seed(0)
  R, S, N_imp, V_dy, V_st = 23, 4, 4, 3, 5
  batch = {"ray_o": torch.randn(R, 3, generator=g), "ray_d": torch.randn(R, 3, generator=g),
           "uv_grid": torch.randn(R, 2, generator=g), "src_cameras": torch.zeros(1, V_dy, 34),
           "static_src_cameras": torch.zeros(1, V_st, 34)}
  jit, u = torch.rand(R, S, generator=g), torch.rand(R, N_imp, generator=g)
  args = (None, None, None, batch, None, None, None, S, None, True, N_imp, False, jit, u)
  whole = _fake_mv_train(*args)
  monkeypatch.setattr(rr, "TRAIN_ROWS_LIMIT", 5 * (S + N_imp) * V_st)  # slices of 5 rays: 5 + 5 + 5 + 5 + 3
  got = rr._render_mv_train_chunked(*args)
  for name, part in whole.items():
    if part is None:
      assert got[name] is None
      continue
    assert list(got[name].keys()) == list(part.keys())
    for k, v in part.items():
      assert got[name][k].shape == v.shape and torch.equal(got[name][k], v), (name, k)
