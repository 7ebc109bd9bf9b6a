"""The float64 reference of the fused per-point stage and the static blending head (tests/point_stage_ref.py)
on the CPU: its bf16 emulation stays close to the exact evaluation, and every planted error would fail the GPU
comparison (tests/test_point_stage_gpu.py) by a wide margin, so its tolerances are not vacuous."""

import pytest
import torch

import point_stage_ref as psr
from dynibar_b200 import synthetic

MARGIN = 3.0  # a planted error must exceed the GPU test's tolerance by this factor on some compared output
R, S, V = 12, 16, 8


@pytest.fixture(scope="module")
def nets():
  model, _ = synthetic.make_model(64, 0, mono=True, seed=4)
  return {"dynamic": model.net_coarse_dy, "static": model.net_coarse_st}


def _chain(kind, net, mode, plant=None):
  """The three point stages in `mode`, each on the kernel-mode outputs of the stage before it (the inputs the
  kernels read on the GPU)."""
  w = net.state_dict()
  G, nvalid, pts, ray_dir = psr.make_point_inputs(R, S, V=V, seed=5)
  k1 = psr.point1(kind, w, G, S)
  out = dict(psr.point1(kind, w, G, S, mode=mode, plant=plant, g2=k1["g2"]))
  out.update({k: v for k, v in psr.attention(k1["Q"], k1["K"], k1["V"], nvalid, S, mode=mode, plant=plant).items()
              if k != "_mag"})
  ka = psr.attention(k1["Q"], k1["K"], k1["V"], nvalid, S)
  shift = float(net.shift) if kind == "dynamic" else 0.0
  out.update(psr.point2(kind, w, ka["O"], k1["g2"], nvalid, S, pts, ray_dir, shift=shift, mode=mode, plant=plant))
  return out


def _head(net, mode, plant=None):
  inp = psr.make_head_inputs(61, V, seed=6)
  return psr.rgb_head(net.state_dict(), inp["X"], inp["vis2"], inp["ray_diff"], inp["mask_eff"], inp["rgb_in"],
                      inp["GW"], inp["sigma"], mode=mode, plant=plant, mask_proj=inp["mask_proj"])


@pytest.mark.parametrize("kind", ["dynamic", "static"])
def test_kernel_mode_agrees_with_exact_mode(nets, kind):
  """Rounding operands, weights and activations to bf16 (relative error <= 2^-9 each) moves every output by a
  few bf16 ulps of its scale, and the masked outputs not at all."""
  k, e = _chain(kind, nets[kind], "kernel"), _chain(kind, nets[kind], "exact")
  if kind == "static":
    k.update(_head(nets[kind], "kernel"))
    e.update(_head(nets[kind], "exact"))
  moved = set()
  for name in e:
    if name.startswith("_"):  # not an output
      continue
    a, b = k[name], e[name]
    masked = b == -1e9
    assert torch.equal(a[masked], b[masked]), name
    err = (a - b)[~masked].abs().max().item()
    scale = b[~masked].abs().max().item()
    assert err <= 16 * 2 ** -9 * scale, (name, err, scale)
    if err > 0:
      moved.add(name)
  assert moved >= {"g2", "Q", "K", "V", "O"}, moved  # the emulation does round


# plant -> (stage, nets it applies to)
_CASES = [(p, "dynamic") for st in ("attention", "point1", "point2") for p in psr.PLANTS[st]]
_CASES += [(p, "static") for p in psr.PLANTS["attention"] + psr.PLANTS["point2"]
           if p not in ("shift_kept", "dir_sincos", "pts_pe_short")]
_CASES += [(p, "static") for p in psr.PLANTS["rgb_head"]]


def _margin(nets, plant, kind):
  if plant in psr.PLANTS["rgb_head"]:
    ref, got = _head(nets[kind], "kernel"), _head(nets[kind], "kernel", plant)
  else:
    ref, got = _chain(kind, nets[kind], "kernel"), _chain(kind, nets[kind], "kernel", plant)
  ratio = {name: e[1] for name, e in psr.errors(got, ref).items()}
  # The attention plants are also scored on the adversarial inputs of the GPU test (logits in the tens).  Keep
  # that case: on the static net's own chain, whose logits are small, scale_128 and query_ge1 stay below 3x,
  # so test_attention_on_adversarial_inputs is what catches them on the GPU.
  if plant in psr.PLANTS["attention"]:
    Q, K, V_, nvalid = psr.make_attention_inputs(R, S, seed=7)
    ref, got = psr.attention(Q, K, V_, nvalid, S), psr.attention(Q, K, V_, nvalid, S, plant=plant)
    ratio["O (adversarial)"] = psr.errors(got, ref)["O"][1]
  return max(ratio.values()), ratio


@pytest.mark.parametrize("plant,kind", _CASES)
def test_planted_error_exceeds_gpu_tolerance(nets, plant, kind):
  margin, ratio = _margin(nets, plant, kind)
  assert margin >= MARGIN, ratio


def test_smallest_plant_margin(nets, capsys):
  margins = {(p, k): _margin(nets, p, k)[0] for p, k in _CASES}
  (p, k), m = min(margins.items(), key=lambda kv: kv[1])
  with capsys.disabled():
    print("\nsmallest planted-error margin: %.1fx (%s, %s net)" % (m, p, k))
  assert m >= MARGIN
