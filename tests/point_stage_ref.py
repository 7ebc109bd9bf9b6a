"""Float64 reference of the fused per-point stage and the static blending head.

Every bf16 render runs, per net, after the per-view stage (tests/view_stage_ref.py):
  point1    csrc/chains_twin.cu: point1_twin_kernel: geometry_fc, + the sinusoid table (dynamic net), Q | K | V;
  attention csrc/attention_tc.cu (S divides 128) or the SIMT attention_kernel<true> (csrc/nets_f32.cu);
  point2    point2_twin_kernel: fc + residual + LayerNorm, then the density and colour heads (dynamic) or the
            density head and GW, the per-point part of rgb_fc.0 (static);
  rgb_head  rgbhead_twin_kernel (static): the per-view blending head and the masked softmax over views.
Each function below evaluates one stage on the inputs the kernel read (so errors do not compound between
stages), with the oracle's formulas (oracle/dynibar_oracle.py: ray_attention, sinusoid_table, periodic_embed
and the heads of net_dynamic / net_static).  Tensors may live on any device; the arithmetic is float64.

mode="exact" evaluates everything in float64 from the fp32 parameters.  mode="kernel" rounds where the kernels
round (line numbers of chains_twin.cu unless noted):
  - the G operand of geometry_fc.0 is bf16 (the tile image the per-view stage writes);
  - hidden activations that only feed another MMA are handed on as bf16(log2(e) ELU(x)) ("exp2 scale",
    fused_engine.cuh: elu_log2; :293, :472, :475, :509, :177): the producing layer's weights are
    bf16(W log2(e)) and its bias the pair hi = bf16(b log2(e)), lo = bf16(b log2(e) - hi) carried by two
    constant-1 operand columns (fused_engine.cuh: append_layer, :637-673); consumers take bf16(W) (weights x
    ln 2 x log2 e) or, where the operand mixes scales, bf16(W log2(e) ln 2) on the exp2-scale columns (:664-667);
  - g2 = ELU(geometry_fc.2) (+ sinusoid) stays fp32 (the residual, :317-322); its bf16 copy is the operand
    of Q | K | V (:324);
  - Q, K, V are stored as bf16 (:329, :334);
  - attention, tensor-core kernels: the unnormalised probabilities P = bf16(e), e = exp((l - max) / sqrt(32)),
    are the operand of P V, which is divided by the fp32 sum of the unrounded e (attention_tc.cu:175-188,
    :354-366); O is stored as bf16 (attention_tc.cu:218, :394).  The SIMT kernel keeps P in fp32 (online
    softmax, nets_f32.cu: attention_kernel) and stores O as bf16: attention(..., simt=True);
  - LayerNorm statistics without cancellation (the kernel: per half-row one pass shifted by one of its values,
    halves combined pairwise in fp32; here the exact mean and variance), and y is a bf16 operand;
  - PE(pts) (:463) and PE(dir) (:481) are bf16 operands;
  - the blending head reads vis2 and ray_diff as bf16 operand columns (:146) next to the bf16 X image;
  - the density logit, the rgb logits and the blending logit are fp32 dot products of the unrounded hidden
    activations (:194, :504, :520).
Query rows with nvalid <= 1 attend uniformly to every key of their ray: the reference masks query rows, not
keys (mlp_network.py:23-24, :91-94).

`plant` names a deliberate error (PLANTS) used to show that the tolerances of the GPU test would catch it.
"""

import math

import torch
import torch.nn.functional as F

from oracle import dynibar_oracle as O

LOG2E, LN2 = 1.0 / math.log(2.0), math.log(2.0)
_LOG2E_F, _LN2_F = torch.tensor(LOG2E, dtype=torch.float32), torch.tensor(LN2, dtype=torch.float32)

# Planted errors (tests/test_point_stage_reference_cpu.py), by the stage they are planted in.  Each must move
# at least one compared output of that stage by at least 3x its tolerance.
PLANTS = {
    "attention": (
        "scale_128",       # logits scaled by 1/sqrt(128) instead of 1/sqrt(32)
        "key_mask",        # keys masked instead of query rows
        "query_ge1",       # query rows kept at nvalid >= 1 instead of > 1
        "neighbor_keys",   # the keys (and values) of the neighbouring ray attended too
        "head_shift",      # head h's probabilities applied to head h+1's values
    ),
    "point1": (
        "sinusoid_next",   # dynamic net: sinusoid row s+1 added to g2
    ),
    "point2": (
        "no_residual",     # residual g2 dropped before the LayerNorm
        "shift_kept",      # dynamic net: sigma - shift not subtracted
        "dir_sincos",      # dynamic net: sin and cos swapped in PE(dir)
        "pts_pe_short",    # dynamic net: PE(pts) with one frequency fewer
        "sigma_nv2",       # sigma masked at nvalid < 2 instead of < 1
    ),
    "rgb_head": (
        "rd_rotate",       # ray_diff columns rotated in rgb_fc.0
        "no_vis2",         # vis2 omitted from rgb_fc.0
        "proj_mask",       # the projector mask used instead of mask_eff
        "all_masked_zero", # a point with every view masked blended to 0 instead of uniformly
        "bias_twice",      # the rgb_fc.0 bias added in both GW and the per-view part
    ),
}

# Tolerances of the GPU comparison, per output: (atol, atol of the "hot" case, ulps or rtol).
#   bf16 outputs (Q, K, V, O):       |got - ref| <= atol + ulps * ulp_bf16(max(|ref|, |got|)) (+ MAG term)
#   fp32 outputs (the rest):         |got - ref| <= atol + rtol * |ref|
# The ulps / rtol term covers the fp32-versus-float64 summation order of the output itself; atol covers bf16
# rounding flips of operands upstream in the stage (a flipped bf16 activation moves the next layer by one
# ulp times a weight).  The hot case (w_qs / w_ks x 4 and the per-point heads' weights x 3) has larger gains.
# Each atol is 1.5 - 3x the largest error measured on an H100, the first over the GPU test's ordinary cases
# (including the LayerNorm-offset and many-tile cases, whose activations are the largest), the second over
# its hot cases only; so a hot atol can be the smaller one where the hot cases' values are smaller.
BF16_OUTPUTS = ("Q", "K", "V", "O")
# Where a sum cancels (the LayerNorm-offset case: g2 is large, V nearly centred), its error scales with the sum
# of the magnitudes of its terms, reference "_mag", rather than with the result: Q, K, V: sum_k |x_k W_nk|
# (the tensor cores' fp32 accumulation); O: sum_j p_j |V_j| (bf16 rounding of the probabilities p).  The
# bound adds MAG[name] * _mag, each coefficient 1.5 - 3x the largest ratio measured on an H100.
MAG = {"Q": 5e-8, "K": 5e-8, "V": 5e-8, "O": 2.0 ** -9}
TOL = {
    "g2": (6e-4, 4e-4, 1e-5),
    "Q": (0.0, 0.0, 1.0),
    "K": (0.0, 0.0, 1.0),
    "V": (0.0, 0.0, 1.0),
    "O": (0.0, 0.0, 1.0),
    "sigma": (1.2e-3, 5e-2, 1e-5),
    "rgb": (4e-4, 1e-2, 1e-5),
    "GW": (2e-3, 3e-3, 1e-5),
    "blend": (1e-5, 6e-4, 1e-5),
}


def bf16(x):
  return x.to(torch.bfloat16).to(torch.float64)


def ulp_bf16(x):
  """One bf16 ulp of x (0 at 0)."""
  m, e = torch.frexp(x.double())
  return torch.where(m != 0, torch.ldexp(torch.ones_like(m), e - 8), torch.zeros_like(m))


class _Units(object):
  """Operand and weight rounding of one mode."""

  def __init__(self, w, mode, device):
    assert mode in ("kernel", "exact")
    self.k = mode == "kernel"
    self.w = w
    self.dev = device

  def p(self, name):
    """fp32 parameter as float64."""
    return self.w[name].detach().to(self.dev, torch.float64)

  def r(self, x):
    """A bf16 operand."""
    return bf16(x) if self.k else x

  def W(self, name, scale=None, colscale=None, cols=None):
    """Weight image: bf16(fp32(W scale) colscale) as append_layer computes it (scale, colscale fp32)."""
    W = self.w[name].detach().to(self.dev, torch.float32)
    if cols is not None:
      W = W[:, cols]
    if not self.k:
      W = W.double()
      return W * (LOG2E if scale == "log2e" else 1.0) * (1.0 if colscale is None else colscale.to(self.dev, torch.float64))
    if scale == "log2e":
      W = W * _LOG2E_F.to(self.dev)
    if colscale is not None:
      W = W * colscale.to(self.dev, torch.float32)
    return bf16(W)

  def b(self, name, scale=None):
    """Folded bias: the hi / lo bf16 pair of fp32(b scale)."""
    b = self.w[name].detach().to(self.dev, torch.float32)
    if not self.k:
      return b.double() * (LOG2E if scale == "log2e" else 1.0)
    if scale == "log2e":
      b = b * _LOG2E_F.to(self.dev)
    hi = b.to(torch.bfloat16).float()
    return hi.double() + bf16(b - hi)


def elu_log2(x2):
  """log2(e) ELU(x) from x2 = log2(e) x (fused_engine.cuh: elu_log2)."""
  return torch.where(x2 > 0, x2, LOG2E * torch.expm1(x2 * LN2))


def elu_from_log2(x2):
  return torch.where(x2 > 0, x2 * LN2, torch.expm1(x2 * LN2))


def _lin(x, W, b=None):
  y = x @ W.t()
  return y if b is None else y + b


def point1(kind, w, G, S, mode="kernel", plant=None, g2=None):
  """point1_twin_kernel: G [P,>=257] (pooled mean | variance | mean weight) -> g2 [P,128] fp32 and Q, K, V
  [P,128].  Q, K, V are computed from `g2` when given (the g2 the kernel wrote), else from this g2."""
  u = _Units(w, mode, G.device)
  G = G.double()[:, :257]
  h = u.r(elu_log2(_lin(u.r(G), u.W("geometry_fc.0.weight", "log2e"), u.b("geometry_fc.0.bias", "log2e"))))
  g = elu_from_log2(_lin(h, u.W("geometry_fc.2.weight"), u.b("geometry_fc.2.bias", "log2e")))
  if kind == "dynamic":
    s = torch.arange(G.shape[0], device=G.device) % S
    if plant == "sinusoid_next":
      s = s + 1
    g = g + O.sinusoid_table(S + 1).to(G.device, torch.float64)[s]
  x = u.r(g if g2 is None else g2.double())
  out = {"g2": g, "_mag": {}}
  for n, k in (("Q", "w_qs"), ("K", "w_ks"), ("V", "w_vs")):
    W = u.W("ray_attention.%s.weight" % k)
    out[n] = u.r(_lin(x, W))
    out["_mag"][n] = _lin(x.abs(), W.abs())  # sum_k |x_k W_nk|: the scale of the fp32 accumulation error
  return out


def attention(Q, K, V, nvalid, S, mode="kernel", simt=False, plant=None):
  """Ray-transformer attention of R = P / S rays: Q, K, V [P,128] (bf16 values), nvalid [P] -> O [P,128]."""
  P = Q.shape[0]
  R = P // S
  sh = lambda t: t.double().reshape(R, S, 4, 32).transpose(1, 2)  # [R,4,S,32]
  q, k, v = sh(Q), sh(K), sh(V)
  nv = nvalid.double().reshape(R, S)
  if plant == "neighbor_keys":
    k = torch.cat([k, k.roll(-1, 0)], 2)
    v = torch.cat([v, v.roll(-1, 0)], 2)
  if plant == "head_shift":
    v = v.roll(-1, 1)
  l = q @ k.transpose(2, 3) / math.sqrt(128.0 if plant == "scale_128" else 32.0)  # [R,4,S,keys]
  valid = nv >= 1 if plant == "query_ge1" else nv > 1
  if plant == "key_mask":
    kv = valid.repeat(1, 2) if plant == "neighbor_keys" else valid
    l = l.masked_fill(~kv[:, None, None, :], -1e9)
  else:
    l = l.masked_fill(~valid[:, None, :, None], -1e9)
  e = torch.exp(l - l.amax(-1, keepdim=True))
  den = e.sum(-1, keepdim=True)
  if mode == "kernel" and not simt:
    o = (bf16(e) @ v) / den
  else:
    o = (e / den) @ v
  o = o.transpose(1, 2).reshape(P, 128)
  mag = ((e / den) @ v.abs()).transpose(1, 2).reshape(P, 128)
  return {"O": bf16(o) if mode == "kernel" else o, "_mag": {"O": mag}}


def point2(kind, w, O_, g2, nvalid, S, pts=None, ray_dir=None, shift=0.0, mode="kernel", plant=None):
  """point2_twin_kernel: O [P,128] (bf16 values), g2 [P,128], nvalid [P] -> dynamic: rgb [P,3] and sigma [P]
  (raw = [rgb, sigma - shift], 0 / -1e9 where no view is valid); static: GW [P,128] and sigma [P]."""
  u = _Units(w, mode, O_.device)
  nv = nvalid.double()
  x = _lin(u.r(O_.double()), u.W("ray_attention.fc.weight"))
  if plant != "no_residual":
    x = x + g2.double()
  mean = x.mean(-1, keepdim=True)
  var = ((x - mean) ** 2).mean(-1, keepdim=True)
  y = (x - mean) / torch.sqrt(var + 1e-6) * u.p("ray_attention.layer_norm.weight") + u.p("ray_attention.layer_norm.bias")
  y = u.r(y)
  none = nv < (2 if plant == "sigma_nv2" else 1)
  sig_w = u.p("out_geometry_fc.2.weight")[0]
  sig_b = u.p("out_geometry_fc.2.bias")[0]
  if kind == "static":
    a = _lin(y, u.W("out_geometry_fc.0.weight", "log2e"), u.b("out_geometry_fc.0.bias", "log2e"))
    sigma = (elu_log2(a) * LN2) @ sig_w + sig_b
    GW = _lin(y, u.W("rgb_fc.0.weight", cols=slice(0, 128)), u.b("rgb_fc.0.bias"))
    return {"GW": GW, "sigma": sigma.masked_fill(none, -1e9)}
  pe = O.periodic_embed(pts.double(), 5)
  if plant == "pts_pe_short":
    pe = pe.clone()
    pe[:, [3 + 12, 3 + 13, 3 + 14, 18 + 12, 18 + 13, 18 + 14]] = 0  # the 2^4 cos and sin columns
  h = u.r(elu_log2(_lin(torch.cat([y, u.r(pe)], -1), u.W("ref_pts_fc.0.weight", "log2e"),
                        u.b("ref_pts_fc.0.bias", "log2e"))))
  g4 = u.r(elu_log2(_lin(h, u.W("ref_pts_fc.2.weight"), u.b("ref_pts_fc.2.bias", "log2e"))))
  ln2 = torch.full((128,), float(_LN2_F))
  a = _lin(g4, u.W("out_geometry_fc.0.weight", "log2e", ln2), u.b("out_geometry_fc.0.bias", "log2e"))
  sigma = (elu_log2(a) * LN2) @ sig_w + sig_b
  if plant != "shift_kept":
    sigma = sigma - shift
  rd = ray_dir.double()[torch.arange(O_.shape[0], device=O_.device) // S]
  pd = O.periodic_embed(rd, 4)
  if plant == "dir_sincos":
    pd = torch.cat([pd[:, :3], pd[:, 15:27], pd[:, 3:15]], -1)
  cs = torch.ones(155)
  cs[:128] = float(_LN2_F)
  h = _lin(torch.cat([g4, u.r(pd)], -1), u.W("rgb_fc.0.weight", "log2e", cs), u.b("rgb_fc.0.bias", "log2e"))
  h = u.r(elu_log2(h))
  a = _lin(h, u.W("rgb_fc.2.weight"), u.b("rgb_fc.2.bias", "log2e"))
  rgb = torch.sigmoid((elu_log2(a) * LN2) @ u.p("rgb_fc.4.weight").t() + u.p("rgb_fc.4.bias"))
  return {"rgb": rgb.masked_fill(none[:, None], 0.0), "sigma": sigma.masked_fill(none, -1e9)}


def rgb_head(w, X, vis2, ray_diff, mask_eff, rgb_in, GW, sigma, mode="kernel", plant=None, mask_proj=None):
  """rgbhead_twin_kernel: X [P,V,128] (bf16 values), vis2, mask_eff [P,V], ray_diff [P,V,4], rgb_in [P,V,3],
  GW [P,128], sigma [P] -> blend [P,3] (raw = [blend, sigma]).  mask_proj: for the plant "proj_mask"."""
  u = _Units(w, mode, X.device)
  rd = ray_diff.double()
  if plant == "rd_rotate":
    rd = rd[..., [1, 2, 3, 0]]
  v2 = vis2.double()
  if plant == "no_vis2":
    v2 = torch.zeros_like(v2)
  op = torch.cat([u.r(X.double()), u.r(v2[..., None]), u.r(rd)], -1)  # [P,V,133]
  a = _lin(op, u.W("rgb_fc.0.weight", "log2e", cols=slice(128, 261)))
  if plant == "bias_twice":
    a = a + u.b("rgb_fc.0.bias", "log2e")
  h = u.r(elu_log2(GW.double()[:, None] * LOG2E + a))
  a = _lin(h, u.W("rgb_fc.2.weight"), u.b("rgb_fc.2.bias", "log2e"))
  logit = (elu_log2(a) * LN2) @ u.p("rgb_fc.4.weight")[0] + u.p("rgb_fc.4.bias")[0]
  mk = (mask_proj if plant == "proj_mask" else mask_eff).double()
  blend = torch.softmax(logit.masked_fill(mk == 0, -1e9), -1)
  if plant == "all_masked_zero":
    blend = blend * (mk.sum(-1, keepdim=True) > 0)
  return {"blend": (blend[..., None] * rgb_in.double()).sum(1), "sigma": sigma.double()}


def errors(got, ref, hot=False, keep=None):
  """Per output of `ref`: (max |got - ref|, max |got - ref| / tolerance, max error beyond the ulps / rtol and
  MAG terms, which atol covers, max error beyond the ulps term per unit of "_mag").  keep: rows to compare (all when None).  Where the reference is masked (sigma
  -1e9, and rgb 0, which a sigmoid never gives) the output must be exactly the masked value."""
  out = {}
  mags = ref.get("_mag", {})
  for name, b in ref.items():
    if name.startswith("_"):
      continue
    atol = TOL[name][1 if hot else 0]
    a, b = got[name].double().to(b.device), b.double()
    mag = mags[name].double() if name in mags else torch.zeros_like(b)
    if keep is not None:
      a, b, mag = a[keep], b[keep], mag[keep]
    if b.numel() == 0:
      out[name] = (0.0, 0.0, 0.0, 0.0)
      continue
    err = (a - b).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, float("inf")), err)
    if name in BF16_OUTPUTS:  # a rounding flip at a binade edge is one ulp of the larger value
      rel = TOL[name][2] * ulp_bf16(torch.maximum(b.abs(), torch.where(torch.isfinite(a), a.abs(), 0.0)))
    else:
      rel = TOL[name][2] * b.abs()
    mc = MAG.get(name, 0.0)
    bound = atol + rel + mc * mag
    masked = (b == -1e9) | ((b == 0) if name == "rgb" else torch.zeros_like(b, dtype=torch.bool))
    err = torch.where(masked, torch.where(a == b, 0.0, float("inf")), err)
    ratio = err / bound
    excess = torch.where(masked, 0.0, err - rel - mc * mag)
    per_mag = torch.where(masked | (mag == 0), 0.0, (err - rel) / mag.clamp(min=1e-300))
    out[name] = (float(torch.where(masked, 0.0, err).max()), float(ratio.max()), float(excess.max()),
                 float(per_mag.max()))
  return out


def make_point_inputs(R, S, V=8, seed=0, g_scale=1.0):
  """Seeded per-point stage inputs: G [P,272] (bf16 values; mean, variance and mean-weight blocks of
  realistic size, the bias columns 264, 265 = 1), nvalid [P] with points of 0, 1, 2 and V valid views, rays
  whose queries are all invalid (nvalid <= 1) and rays with a single valid query, pts [P,3], ray_dir [R,3]."""
  g = torch.Generator().manual_seed(seed)
  P = R * S
  G = torch.zeros(P, 272)
  G[:, :128] = torch.randn(P, 128, generator=g) * 0.5 * g_scale
  G[:, 128:256] = torch.randn(P, 128, generator=g).abs() * 0.2 * g_scale
  G[:, 256] = torch.rand(P, generator=g) / V
  G[:, 264:266] = 1.0
  G = G.to(torch.bfloat16).float()
  choices = torch.tensor([0.0, 1.0, 2.0, float(V)])
  nvalid = choices[torch.randint(0, 4, (P,), generator=g)].reshape(R, S)
  if R >= 3:
    nvalid[1] = torch.randint(0, 2, (S,), generator=g).float()  # no valid query
    nvalid[2] = torch.randint(0, 2, (S,), generator=g).float()  # exactly one valid query
    nvalid[2, S // 2] = float(V)
  pts = torch.randn(P, 3, generator=g) * 2
  ray_dir = F.normalize(torch.randn(R, 3, generator=g), dim=-1)
  return G, nvalid.reshape(P).contiguous(), pts, ray_dir


def make_attention_inputs(R, S, seed=0):
  """Adversarial attention inputs (bf16 values): Q, K with logits / sqrt(32) in the tens, keys tied in pairs,
  constant query rows, rays whose values are constant over the keys; nvalid as make_point_inputs."""
  g = torch.Generator().manual_seed(seed)
  P = R * S
  Q = torch.randn(P, 128, generator=g) * 4.0
  K = torch.randn(R, S, 128, generator=g) * 4.0
  V = torch.randn(R, S, 128, generator=g)
  Q[5::7] = 2.5                          # constant query rows
  K[:, 1::2] = K[:, 0::2][:, : S // 2]   # ties: key 2j+1 = key 2j
  V[0::3] = V[0::3, :1]                  # values constant over the keys of every third ray
  _, nvalid, _, _ = make_point_inputs(R, S, seed=seed)
  bf = lambda t: t.reshape(P, 128).to(torch.bfloat16).float().contiguous()
  return bf(Q), bf(K), bf(V), nvalid


def make_head_inputs(P, V, seed=0):
  """Seeded blending-head inputs: X [P,V,128] (bf16 values), vis2, mask_proj, mask_eff [P,V], ray_diff
  [P,V,4], rgb_in [P,V,3], GW [P,128], sigma [P].  mask_eff drops some projector-valid views (as mask_rgb
  does); there are points with every view masked and points with one valid view."""
  g = torch.Generator().manual_seed(seed)
  X = (torch.randn(P, V, 128, generator=g) * 0.7).to(torch.bfloat16).float()
  mask_proj = (torch.rand(P, V, generator=g) < 0.8).float()
  mask_eff = mask_proj * (torch.rand(P, V, generator=g) < 0.8).float()
  mask_eff[0::7] = 0.0                     # every view masked
  mask_eff[3::7] = 0.0
  mask_eff[3::7, V // 2] = 1.0             # one valid view
  vis2 = torch.rand(P, V, generator=g) * mask_eff
  d = F.normalize(torch.randn(P, V, 3, generator=g), dim=-1) * 0.3
  ray_diff = torch.cat([d, 1.0 - torch.rand(P, V, 1, generator=g) * 0.5], -1)
  rgb_in = torch.rand(P, V, 3, generator=g)
  GW = torch.randn(P, 128, generator=g) * 0.5
  sigma = torch.randn(P, generator=g)
  sigma[0::11] = -1e9
  return dict(X=X, vis2=vis2, mask_proj=mask_proj, mask_eff=mask_eff, ray_diff=ray_diff.contiguous(),
              rgb_in=rgb_in, GW=GW, sigma=sigma)


def scale_weights(net, qk=1.0, heads=1.0, geo2_bias=0.0):
  """In place: w_qs / w_ks x qk; the per-point heads (ref_pts_fc, out_geometry_fc, rgb_fc) x heads;
  geometry_fc.2 bias + geo2_bias, with the rows of w_vs centred when geo2_bias is set, so that the offset
  reaches the LayerNorm input x = fc(O) + g2 through the residual only and x's mean dwarfs its spread."""
  with torch.no_grad():
    for name, p in net.named_parameters():
      if name in ("ray_attention.w_qs.weight", "ray_attention.w_ks.weight"):
        p.mul_(qk)
      if name.startswith(("ref_pts_fc.", "out_geometry_fc.", "rgb_fc.")) and name.endswith(".weight"):
        p.mul_(heads)
      if name == "geometry_fc.2.bias":
        p.add_(geo2_bias)
      if name == "ray_attention.w_vs.weight" and geo2_bias:
        p.sub_(p.mean(1, keepdim=True))
