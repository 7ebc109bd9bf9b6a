"""The fused per-point stage (point1, the ray-transformer attention, point2) and the static blending head against
a float64 reference that rounds to bf16 where the kernels do (tests/point_stage_ref.py, mode="kernel").

dyn_debug_point_chain runs point1 -> attention -> point2 on caller-provided pooled features and returns what
each stage wrote (g2, Q, K, V, O and the heads' outputs), so every stage is compared on the inputs it actually
read.  dyn_debug_attention runs the product's attention dispatch on caller-provided Q, K, V (adversarial logits,
ties, constant rows); dyn_debug_rgb_head runs the blending head on per-view rows.  The sample counts reach every
attention kernel a render can run: the twin kernels (S = 64, 128), attention_tc_kernel<false> (S = 1 .. 32
dividing 128) and the SIMT kernel (20, 48, 192, 512).  The reference is evaluated on the GPU in float64.
"""

import pytest
import torch

import point_stage_ref as psr
import view_stage_ref as vr
from dynibar_b200 import _lib, synthetic, weights

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (S, R, variant): ragged R everywhere (37 rays at S = 64 leave one ray in the last tile); 1301 x 64 and
# 701 x 128 give every persistent CTA several tiles (the attention kernels' next-tile prefetch)
CHAIN_CASES = [(S, 37, "") for S in (1, 8, 16, 32, 64, 128, 20, 48, 192)] + [
    (512, 9, ""), (64, 1301, ""), (128, 701, ""),
    # w_qs / w_ks x 4 (the softmax saturates), per-point heads x 3
    (64, 37, "hot"), (16, 37, "hot"), (48, 37, "hot"),
    # geometry_fc.2 bias + 16 (w_vs rows centred): the LayerNorm input's mean dwarfs its spread, which
    # stresses the single-pass variance
    (64, 37, "ln16"), (20, 37, "ln16"),
]


def _tc(S):
  return S >= 1 and S <= 128 and 128 % S == 0


def _net(kind, variant=""):
  model, _ = synthetic.make_model(64, 0, mono=True, seed=4)
  net = model.net_coarse_dy if kind == "dynamic" else model.net_coarse_st
  if variant == "hot":
    psr.scale_weights(net, qk=4.0, heads=3.0)
  if variant == "ln16":
    psr.scale_weights(net, geo2_bias=16.0)
  return net.to(DEV)


def _nan(*shape):
  return torch.full(shape, float("nan"), device=DEV)


def run_chain(net, kind, G, nvalid, pts, ray_dir, R, S):
  """dyn_debug_point_chain -> dict of CUDA tensors: g2, Q, K, V, O and out_a, out_b."""
  P = R * S
  packed = weights.packed_of(net, torch.device(DEV))
  d = lambda x: x.to(DEV).contiguous()
  Gd, nvd, ptd, rdd = d(G), d(nvalid), d(pts), d(ray_dir)
  out = {k: _nan(P, 128) for k in ("g2", "Q", "K", "V", "O")}
  out["out_a"] = _nan(P, 128 if kind == "static" else 4)
  out["out_b"] = _nan(P)
  pws = torch.zeros(S * 128, device=DEV)
  _lib.check(_lib.lib.dyn_debug_point_chain(
      packed.handle, Gd.data_ptr(), nvd.data_ptr(), ptd.data_ptr(), rdd.data_ptr(), R, S,
      *[out[k].data_ptr() for k in ("g2", "Q", "K", "V", "O", "out_a", "out_b")], pws.data_ptr(), _lib.stream()))
  torch.cuda.synchronize()
  return out


def compare_chain(kind, S, R, variant):
  """One chain case -> {stage: errors dict} and facts."""
  net = _net(kind, variant)
  w = net.state_dict()
  G, nvalid, pts, ray_dir = psr.make_point_inputs(R, S, seed=S + R)
  got = run_chain(net, kind, G, nvalid, pts, ray_dir, R, S)
  G, nvalid, pts, ray_dir = (t.to(DEV) for t in (G, nvalid, pts, ray_dir))
  hot = variant == "hot"
  errs = {}
  ref1 = psr.point1(kind, w, G, S, g2=got["g2"])
  errs["point1"] = psr.errors(got, ref1, hot)
  ref_a = psr.attention(got["Q"], got["K"], got["V"], nvalid, S, simt=not _tc(S))
  errs["attention"] = psr.errors(got, ref_a, hot)
  ref2 = psr.point2(kind, w, got["O"], got["g2"], nvalid, S, pts, ray_dir, shift=float(net.shift) if kind == "dynamic" else 0.0)
  if kind == "dynamic":
    g2out = {"rgb": got["out_a"][:, :3], "sigma": got["out_a"][:, 3]}
  else:
    g2out = {"GW": got["out_a"], "sigma": got["out_b"]}
  errs["point2"] = psr.errors(g2out, ref2, hot)
  facts = {"finite": all(bool(torch.isfinite(got[k]).all()) for k in ("g2", "Q", "K", "V", "O")),
           "nvalid_classes": sorted(set(nvalid.tolist())),
           "masked_sigma": int((ref2["sigma"] == -1e9).sum())}
  # the LayerNorm input x = fc(O) + g2: how far its mean stands off against its spread
  x = psr.bf16(got["O"].double()) @ psr.bf16(w["ray_attention.fc.weight"].double()).t() + got["g2"].double()
  facts["ln_mean_over_std"] = float((x.mean(-1).abs() / x.std(-1, unbiased=False)).median())
  return errs, facts


@pytest.mark.parametrize("kind", ["dynamic", "static"])
@pytest.mark.parametrize("S,R,variant", CHAIN_CASES)
def test_point_stage_matches_reference(kind, S, R, variant):
  errs, facts = compare_chain(kind, S, R, variant)
  print(kind, S, R, variant, errs)
  assert facts["finite"], facts
  assert {0.0, 1.0, 2.0, 8.0} <= set(facts["nvalid_classes"]) and facts["masked_sigma"] > 0, facts
  if variant == "ln16":  # the single-pass variance E[x^2] - mean^2 cancels at least 100:1
    assert facts["ln_mean_over_std"] >= 10, facts
  bad = {(st, k): v for st, e in errs.items() for k, v in e.items() if v[1] > 1.0}
  assert not bad, "outputs out of tolerance ((stage, output): (max |err|, err / tol)): %s" % bad


# adversarial attention inputs on dyn_debug_attention: (S, R)
ATTN_CASES = [(1, 37), (8, 37), (32, 37), (64, 37), (128, 21), (20, 37), (48, 37), (192, 5)]


def run_attention(Q, K, V, nvalid, R, S):
  d = lambda x: x.to(DEV).contiguous()
  Qd, Kd, Vd, nvd = d(Q), d(K), d(V), d(nvalid)
  O = _nan(R * S, 128)
  rc = _lib.lib.dyn_debug_attention(Qd.data_ptr(), Kd.data_ptr(), Vd.data_ptr(), nvd.data_ptr(), R, S, O.data_ptr(),
                                    _lib.stream())
  torch.cuda.synchronize()
  return rc, O


@pytest.mark.parametrize("S,R", ATTN_CASES)
def test_attention_on_adversarial_inputs(S, R):
  Q, K, V, nvalid = psr.make_attention_inputs(R, S, seed=100 + S)
  rc, O = run_attention(Q, K, V, nvalid, R, S)
  _lib.check(rc)
  ref = psr.attention(Q.to(DEV), K.to(DEV), V.to(DEV), nvalid.to(DEV), S, simt=not _tc(S))
  errs = psr.errors({"O": O}, ref)
  print(S, R, errs)
  assert errs["O"][1] <= 1.0, errs


def test_simt_attention_rejects_samples_beyond_its_block_limit():
  """S = 1024 needs 1024 threads per block, more than the SIMT attention kernels can launch with their register
  counts: both the fused and the staged path fail with DYN_E_INVALID before launching anything."""
  R, S, V = 1, 1024, 1
  P = R * S
  e = lambda *shape: torch.empty(*shape, device=DEV)  # no fill kernel
  Q, O, nvalid = e(P, 128), e(P, 128), e(P)
  rc = _lib.lib.dyn_debug_attention(Q.data_ptr(), Q.data_ptr(), Q.data_ptr(), nvalid.data_ptr(), R, S, O.data_ptr(),
                                    _lib.stream())
  msg = _lib.lib.dyn_last_error().decode()
  assert rc == -1 and "SIMT attention kernel supports S <= " in msg, (rc, msg)
  limit = int(msg.split("S <= ")[1].split()[0])
  assert 512 <= limit < 1024, msg  # config-4's fine pass (192) and the 512-sample case above must run
  model, _ = synthetic.make_model(64, 0, mono=True, seed=4)
  net = weights.PackedNet(model.net_coarse_dy, torch.device(DEV), level=0)  # fp32 parameters only: no packing kernels
  nbytes = _lib.lib.dyn_net_workspace_bytes(_lib.NET_DYNAMIC, R, S, V)
  ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
  pts, feat, rd, mask, raw = e(P, 3), e(P, V, 35), e(R, 3), e(P, V), e(P, 4)
  rc = _lib.lib.dyn_net_dynamic(net.handle, pts.data_ptr(), feat.data_ptr(), rd.data_ptr(), mask.data_ptr(), 0.0, R,
                                S, V, raw.data_ptr(), ws.data_ptr(), nbytes, _lib.PREC_FP32, _lib.stream())
  msg = _lib.lib.dyn_last_error().decode()
  assert rc == -1 and "SIMT attention kernel supports S <= " in msg, (rc, msg)


# blending head: (V, P, variant); P * VP is not a multiple of 128 anywhere
HEAD_CASES = [(1, 185, ""), (2, 185, ""), (7, 185, ""), (8, 185, ""), (9, 93, ""), (11, 93, ""), (16, 93, ""),
              (8, 4001, ""), (8, 185, "hot"), (16, 93, "hot")]


def run_rgb_head(net, inp, P, V):
  packed = weights.packed_of(net, torch.device(DEV))
  d = {k: v.to(DEV).contiguous() for k, v in inp.items()}
  raw = _nan(P, 4)
  _lib.check(_lib.lib.dyn_debug_rgb_head(packed.handle, *[d[k].data_ptr() for k in (
      "X", "vis2", "ray_diff", "mask_eff", "rgb_in", "GW", "sigma")], P, V, raw.data_ptr(), _lib.stream()))
  torch.cuda.synchronize()
  return raw


@pytest.mark.parametrize("V,P,variant", HEAD_CASES)
def test_blending_head_matches_reference(V, P, variant):
  net = _net("static", variant)
  inp = psr.make_head_inputs(P, V, seed=V * 1000 + P)
  raw = run_rgb_head(net, inp, P, V)
  d = {k: v.to(DEV) for k, v in inp.items()}
  ref = psr.rgb_head(net.state_dict(), d["X"], d["vis2"], d["ray_diff"], d["mask_eff"], d["rgb_in"], d["GW"],
                     d["sigma"])
  errs = psr.errors({"blend": raw[:, :3], "sigma": raw[:, 3]}, ref, hot=variant == "hot")
  print(V, P, variant, errs)
  assert torch.equal(raw[:, 3], d["sigma"]), "sigma is not passed through"
  assert errs["blend"][1] <= 1.0, errs
  # the inputs hold points with every view masked and with one valid view, and views mask_rgb would reject
  assert (inp["mask_eff"].sum(1) == 0).any() and (inp["mask_eff"].sum(1) == 1).any() and (inp["mask_eff"] != inp["mask_proj"]).any()


# scenes of tests/view_stage_ref.make_case (as in test_view_stage_gpu.py): the benchmark shape, a launch of two
# internal chunks (net_rows_per_chunk(128, 16) = 2048 rays), exact-black sources under mask_rgb, virtual views
WIRING_CASES = {
    "bench": dict(V=8, rays=300, S=64, seed=29),
    "two_chunks": dict(V=16, rays=2050, S=128, seed=30, H=48, W=64),
    "mask_rgb": dict(V=8, rays=96, S=16, seed=32, mask_rgb=1, black=True, stress=True),
    "vv_far": dict(V=10, rays=60, S=32, seed=35, num_vv=3, far=30.0),
}


@pytest.mark.parametrize("kind", ["static", "dynamic"])
@pytest.mark.parametrize("case", list(WIRING_CASES))
def test_hooks_reproduce_fused_render_bit_exactly(case, kind):
  """The captured per-view outputs of a fused render, run through dyn_debug_point_chain (and, for the static
  net, dyn_debug_rgb_head), give the render's raw bit for bit, across internal chunk boundaries too: the
  hooks run the product's kernels on the product's data layouts."""
  from dynibar_b200 import render_ray as rr
  nets, st, dy = vr.make_case(**WIRING_CASES[case])
  sc = st if kind == "static" else dy
  net = nets[kind].to(DEV)
  d = lambda t: t.to(DEV)
  V = sc["src_cams"].shape[0]
  P, S = sc["pts"].shape[0], sc["S"]
  R = P // S
  cap = {"G": _nan(P, vr.GCOLS), "nvalid": _nan(P), "X": _nan(P, V, 128), "vis2": _nan(P, V),
         "mask_eff": _nan(P, V), "ray_diff": _nan(P, V, 4), "rgb_in": _nan(P, V, 3)}
  order = ("G", "nvalid", "X", "vis2", "mask_eff", "ray_diff", "rgb_in")
  pts = d(sc["pts"]).reshape(R, S, 3)
  cams, rgbs = d(sc["src_cams"])[None], d(sc["src_rgbs"])[None]
  feat = rr.featmaps_channels_last(d(sc["featmaps"]))
  ray_dir = torch.nn.functional.normalize(d(sc["ray_d"]), dim=-1)
  _lib.lib.dyn_debug_set_view_capture(*[cap[k].data_ptr() for k in order])
  try:
    if kind == "static":
      raw, _ = rr.net_static_fused(net, pts, d(sc["ray_o"]), d(sc["ray_d"]), d(sc["query_cam"])[None], rgbs, cams,
                                   feat)
    else:
      seq = d(sc["pts_seq"]).reshape(V, R, S, 3)
      raw, _ = rr.net_dynamic_fused(net, pts, seq, ray_dir, d(sc["query_cam"])[None], rgbs, cams, feat, sc["time"])
    torch.cuda.synchronize()
  finally:
    _lib.lib.dyn_debug_set_view_capture(None, None, None, None, None, None, None)
  raw = raw.reshape(P, 4)
  got = run_chain(net, kind, cap["G"], cap["nvalid"], pts.reshape(P, 3), ray_dir, R, S)
  if kind == "static":
    hook = run_rgb_head(net, {"X": cap["X"], "vis2": cap["vis2"], "ray_diff": cap["ray_diff"],
                              "mask_eff": cap["mask_eff"], "rgb_in": cap["rgb_in"], "GW": got["out_a"],
                              "sigma": got["out_b"]}, P, V)
  else:
    hook = got["out_a"]
  diff = (hook != raw).any(1)
  assert not diff.any(), "rows differing from the fused render: %d of %d (first %d)" % (
      int(diff.sum()), P, int(torch.nonzero(diff)[0, 0]))

