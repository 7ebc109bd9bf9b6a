"""The float64 reference of the fused per-view stage (tests/view_stage_ref.py) on the CPU: its bf16 emulation
stays close to the exact evaluation, and every planted error of the stage would fail the GPU comparison
(tests/test_view_stage_gpu.py) of the warpgroup kernel, the one every bf16 render runs, by a wide margin, so
its tolerances are not vacuous."""

import pytest
import torch

import view_stage_ref as vr

MARGIN = 3.0  # a planted error must exceed the GPU test's tolerance by this factor on some compared output


@pytest.fixture(scope="module")
def scene():
  # 64 rays x 32 samples, 8 views; exact-black source regions and a stressed rig so that mask_rgb and the
  # anti-alias minimum over views both matter
  return vr.make_case(V=8, rays=64, S=32, seed=3, mask_rgb=1, black=True, stress=True)


@pytest.fixture(scope="module")
def refs(scene):
  nets, st, dy = scene
  out = {}
  for kind, sc in (("static", st), ("dynamic", dy)):
    w = nets[kind].state_dict()
    out[kind] = (w, sc, vr.view_stage(kind, w, sc, mode="kernel"), vr.view_stage(kind, w, sc, mode="exact"))
  return out


@pytest.mark.parametrize("kind", ["static", "dynamic"])
def test_kernel_mode_agrees_with_exact_mode(refs, kind):
  """Rounding the GEMM operands to bf16 (relative error <= 2^-9 each) moves the outputs by a few bf16 ulps of
  their block's scale, and by nothing where the kernel does not round (masks, gathered colours, geometry)."""
  _, _, k, e = refs[kind]
  ck, ce = vr.compared(k, kind), vr.compared(e, kind)
  for name in ("mask_eff", "rgb_in", "ray_diff", "nvalid"):
    if name in ce:
      assert torch.equal(ck[name], ce[name]), name
  assert torch.equal(k["mask_proj"], e["mask_proj"])
  moved = False
  for name in ("G_mean", "G_var", "G_w", "X", "vis2"):
    if name not in ce:
      continue
    err = (ck[name] - ce[name]).abs().max().item()
    scale = ce[name].abs().max().item()
    assert err <= 16 * 2 ** -9 * scale, (name, err, scale)
    moved |= err > 0
  assert moved  # the emulation does round


# plant -> the net it applies to (the others need the static net's inputs or are static-only)
_PLANT_NET = {p: "static" for p in vr.PLANTS}
_PLANT_NET["no_time"] = "dynamic"


@pytest.mark.parametrize("plant", vr.PLANTS)
def test_planted_error_exceeds_gpu_tolerance(refs, plant):
  kind = _PLANT_NET[plant]
  w, sc, k, _ = refs[kind]
  ratio = {name: r for name, (_, r) in vr.errors(vr.view_stage(kind, w, sc, plant=plant), k, kind).items()}
  assert max(ratio.values()) >= MARGIN, ratio


@pytest.mark.parametrize("plant", ["var2_drop", "var2_scale", "vis0_over_V", "var1_drop", "chan_drop",
                                   "view_swap", "W_over_nvalid"])
def test_planted_error_in_dynamic_net_exceeds_gpu_tolerance(refs, plant):
  """The dynamic net's capture has G and nvalid only: the errors both nets can make show there too."""
  w, sc, k, _ = refs["dynamic"]
  ratio = {name: r for name, (_, r) in vr.errors(vr.view_stage("dynamic", w, sc, plant=plant), k, "dynamic").items()}
  assert max(ratio.values()) >= MARGIN, ratio
