"""Float64 reference of the staged training forward and its backward: DynibarDynamic, DynibarStatic, MotionMLP.

The library's training step evaluates each network with the staged kernels of csrc/nets_f32.cu in training mode
(net_dynamic_f32 / net_static_f32 with `train = true`: run_trunk, run_point_tail, the heads) and
motion_train_forward (csrc/motion_train.cu), keeps every activation, and differentiates it in
csrc/nets_train.cu / csrc/motion_train.cu.  This module restates that computation: the glue (poolings, visibility
gating, LayerNorm, attention with the query-row mask quirk, positional encodings, the heads) with the oracle's
formulas (oracle/dynibar_oracle.py) differentiated by torch autograd, and every linear layer through one
autograd Function, _Linear, which mirrors the library's LinArgs / Seg (csrc/linear_f32.cuh): input segments, each
a tensor plus a broadcast divisor, an optional row scale and an activation.  Tensors may live on any device; the
arithmetic is float64.

mode="exact" does all arithmetic in float64: the library's precision "fp32" (every product in fp32 SIMT).
mode="kernel" rounds where precision "bf16" rounds, and nowhere else: a product that dispatch() puts on the tensor
cores multiplies round-to-nearest bf16 copies of both operands (the row-scaled input X rs, the weight, dZ) and
accumulates exactly; every other product, and all the glue, is exact.  The bias is added after the product.

`plant` names a deliberate wiring error (PLANTS, FWD_PLANTS) used to show that the bars of the GPU tests would
catch it.

The same functions state the inference forward (net_*_f32 with `train = false`): its arithmetic is the training
forward's, only its buffers differ (X2 and H3 updated in place, the rays split into internal chunks).
make_forward_case / forward serve that comparison (tests/test_staged_nets_gpu.py).
"""

import math

import torch
import torch.nn.functional as F

from oracle import dynibar_oracle as O

# Planted wiring errors (tests/test_train_stage_reference_cpu.py).  Not among them: dropping the 1-column remainder
# of geometry_fc.0's dIn.  That column, d/dG[:, 256] with G[:, 256] = mean_v vis2 / (sum vis2 + 1e-8) = 1 / V to
# within 1e-8 / sum vis2, reaches no gradient by more than 1e-6 of a bar, so no test can see it.  Each must move at least one compared output of
# the case it is scored on by at least MARGIN times its bar.
PLANTS = (
    "rowscale_dw",      # the row scale dropped from the weight gradient of vis_fc.0 / vis_fc2.0
    "geo0_rem_col0",    # the 1-column remainder of geometry_fc.0's 257-wide dW split taken from column 0 of X
    "skip_dIn_drop",    # columns 256..387 of MotionMLP pts_linears.5's dIn dropped
    "partial_stage",    # the rows of the partial last 64-row stage left out of every tensor-core weight gradient
    "bcast_one",        # a broadcast segment's gradients use the first view's (sample's) dZ, not the group sum
    "bias_P",           # a per-view bias gradient summed over the first P rows instead of all M
    "acc_overwrite",    # out_geometry_fc.0's dIn overwrites dG4 / dG3 instead of adding: rgb_fc.0's share is lost
    "nblock_x",         # the second 128-column N block of a tensor-core dW reads X's first block
)


def bf16(x):
  return x.to(torch.bfloat16).to(x.dtype)


# ---------------------------------------------------------------------------------------------------------------
# Dispatch: which product runs on the tensor cores (bf16 operands) and which in fp32 SIMT.  Every rule of the
# library's bf16 training path is here; if a threshold moves in the library, the GPU test fails and points here.
# ---------------------------------------------------------------------------------------------------------------
def tc_grad_w_ok(out, width, rows):
  """csrc/train_tc.cu: tc_grad_w_ok."""
  return 1 <= out <= 256 and 1 <= width <= 256 and rows >= 2048


def tc_grad_in_ok(out, width, rows):
  """csrc/train_tc.cu: tc_grad_in_ok."""
  return 16 <= width <= 256 and out >= 16 and rows >= 2048


def dispatch(op, net, out, width, rows, layer="", accumulate=False):
  """Column pieces [(c0, c1, on_tensor_cores)] of one product of a layer with `out` outputs, reading `width` input
  columns over `rows` rows, in precision bf16.

  op "fwd"      Y = act(X W^T + b).  Nets: run_lin, csrc/nets_f32.cu:576-580 (M >= 128 and out >= 16).  MotionMLP:
                motion_train_forward, csrc/motion_train.cu:229-234 (pts_linears at N >= 128; coeff_linear SIMT).
  op "grad_w"   dW += dZ^T X over the rows of the segment (group sums first for broadcast segments).  Nets:
                Prod::grad_w, csrc/nets_train.cu:525-538 (split at 256 columns, the remainder dispatched again).
                MotionMLP: csrc/motion_train.cu:248-253 (whole segment).
  op "grad_in"  dIn = dZ W[:, c0:c0+width].  Nets: Prod::grad_in, csrc/nets_train.cu:540-551 (split at 256, the
                remainder dispatched again; an accumulating call, Q|K|V into dG2 :642-644 and out_geometry_fc.0
                into dG4 / dG3 :749, :814, is always SIMT).  MotionMLP: csrc/motion_train.cu:254-262 (above 256
                columns both pieces on the tensor cores or neither).
  """
  if op == "fwd":
    if net == "motion":
      return [(0, width, layer != "coeff_linear" and rows >= 128)]
    return [(0, width, rows >= 128 and out >= 16)]
  ok = tc_grad_w_ok if op == "grad_w" else tc_grad_in_ok
  if op == "grad_in" and accumulate:
    return [(0, width, False)]
  if net == "motion":
    if width <= 256:
      return [(0, width, ok(out, width, rows))]
    both = ok(out, 256, rows) and ok(out, width - 256, rows)
    return [(0, 256, True), (256, width, True)] if both else [(0, width, False)]
  pieces, c0 = [], 0
  while width - c0 > 256 and ok(out, 256, rows):
    pieces.append((c0, c0 + 256, True))
    c0 += 256
  pieces.append((c0, width, ok(out, width - c0, rows)))
  return pieces


class _Spec(object):
  """One layer call: name, net ("dynamic" / "static" / "motion"), broadcast divisors of the segments, activation,
  whether its dIn accumulates, P of a per-view layer (for the plant bias_P), rounding on / off, plant, stats."""

  def __init__(self, name, net, divs, act, acc_in, P, kernel, plant, stats):
    self.name, self.net, self.divs, self.act, self.acc_in = name, net, divs, act, acc_in
    self.P, self.k, self.plant, self.stats = P, kernel, plant, stats


def _act(z, act):
  if act == "elu":
    return F.elu(z)
  if act == "relu":
    return torch.relu(z)
  if act == "sigmoid":
    return torch.sigmoid(z)
  return z


def _act_grad(z, act):
  if act == "elu":
    return torch.where(z > 0, torch.ones_like(z), torch.exp(z))
  if act == "relu":
    return (z > 0).to(z.dtype)
  if act == "sigmoid":
    s = torch.sigmoid(z)
    return s * (1 - s)
  return torch.ones_like(z)


def _grad_w(sp, G, X, out):
  """dW [out, width] = G^T X over the rows of G / X, per dispatch piece."""
  rows, width = X.shape
  res = G.new_zeros(out, width)
  for c0, c1, tc in dispatch("grad_w", sp.net, out, width, rows):
    Gp, Xp = G, X[:, c0:c1]
    if sp.plant == "geo0_rem_col0" and sp.name == "geometry_fc.0" and c0 == 256:
      Xp = X[:, 0:c1 - c0]
    if tc:
      if sp.k:
        Gp, Xp = bf16(Gp), bf16(Xp)
      if sp.plant == "partial_stage" and rows % 64:
        keep = rows - rows % 64
        Gp, Xp = Gp[:keep], Xp[:keep]
      if sp.plant == "nblock_x" and c1 - c0 > 128:
        Xp = torch.cat([Xp[:, :128], Xp[:, :c1 - c0 - 128]], 1)
    res[:, c0:c1] = Gp.t() @ Xp
  return res


def _grad_in(sp, G, W):
  """dIn [rows, width] = G W (W [out, width]), per dispatch piece."""
  out, width = W.shape
  res = G.new_zeros(G.shape[0], width)
  for c0, c1, tc in dispatch("grad_in", sp.net, out, width, G.shape[0], accumulate=sp.acc_in):
    Gp, Wp = G, W[:, c0:c1]
    if tc and sp.k:
      Gp, Wp = bf16(Gp), bf16(Wp)
    res[:, c0:c1] = Gp @ Wp
  return res


class _Linear(torch.autograd.Function):
  """Y = act(cat_i(expand(x_i, div_i)) rs W^T + b) with the library's products in both directions."""

  @staticmethod
  def forward(ctx, sp, W, b, rs, *xs):
    X = torch.cat([x.repeat_interleave(d, 0) if d > 1 else x for x, d in zip(xs, sp.divs)], 1)
    if rs is not None:
      X = X * rs[:, None]
    tc = dispatch("fwd", sp.net, W.shape[0], X.shape[1], X.shape[0], layer=sp.name)[0][2]
    Z = (bf16(X) @ bf16(W).t()) if (tc and sp.k) else X @ W.t()
    if b is not None:
      Z = Z + b
    if sp.act == "relu" and sp.stats is not None:
      # pre-activations within reach of the fp32 / float64 difference: their ReLU may take the other side on the GPU
      Xr, Wr = (bf16(X), bf16(W)) if (tc and sp.k) else (X, W)
      mag = Xr.abs() @ Wr.abs().t() + (b.abs() if b is not None else 0.0)
      near = (Z.abs() <= RELU_NEAR * mag)
      sp.stats[sp.name] = (int(near.sum()), Z.numel())
    ctx.sp = sp
    ctx.save_for_backward(W, rs, Z, *xs)
    return _act(Z, sp.act)

  @staticmethod
  def backward(ctx, dY):
    sp = ctx.sp
    W, rs, Z, *xs = ctx.saved_tensors
    out = W.shape[0]
    dZ = dY * _act_grad(Z, sp.act)
    gW = W.new_zeros(W.shape)
    gx = []
    d_rs = None
    c0 = 0
    for i, (x, d) in enumerate(zip(xs, sp.divs)):
      w = x.shape[1]
      if d > 1:  # broadcast segment: fp32 group sum, then products over the coarser rows
        G = dZ.view(-1, d, out)[:, 0] if sp.plant == "bcast_one" else dZ.view(-1, d, out).sum(1)
      else:
        G = dZ
      Xi = x if (rs is None or (sp.plant == "rowscale_dw" and sp.name in ("vis_fc.0", "vis_fc2.0"))) else x * rs[:, None]
      gW[:, c0:c0 + w] = _grad_w(sp, G, Xi, out)
      g = None
      if ctx.needs_input_grad[4 + i]:
        g = _grad_in(sp, G, W[:, c0:c0 + w])
        if sp.plant == "acc_overwrite" and sp.name == "rgb_fc.0" and i == 0:
          g = torch.zeros_like(g)
        if sp.plant == "skip_dIn_drop" and sp.name == "pts_linears.5" and i == 1:
          g[:, 256 - c0:] = 0.0  # columns 256..387 of the 388-wide product
        if rs is not None:  # rowscale_bwd_kernel: d rs = sum_c dXs x, dx = dXs rs
          d_rs = (g * x).sum(1)
          g = g * rs[:, None]
      gx.append(g)
      c0 += w
    db = None
    if ctx.needs_input_grad[2]:
      db = (dZ[:sp.P] if (sp.plant == "bias_P" and sp.P is not None) else dZ).sum(0)
    return (None, gW, db, d_rs if ctx.needs_input_grad[3] else None) + tuple(gx)


# a ReLU pre-activation counts as "near 0" when |z| <= RELU_NEAR sum_k |x_k W_nk| (+ |b|): about 256 fp32 ulps
# of the accumulation's scale, well beyond the fp32 accumulation error of a 388-term product
RELU_NEAR = 2.0 ** -16


class _Net(object):
  def __init__(self, w, net, mode, plant, stats=None):
    assert mode in ("exact", "kernel")
    self.w, self.net, self.k, self.plant, self.stats = w, net, mode == "kernel", plant, stats

  def lin(self, name, segs, act, rs=None, acc_in=False, P=None):
    sp = _Spec(name, self.net, tuple(d for _, d in segs), act, acc_in, P, self.k, self.plant, self.stats)
    return _Linear.apply(sp, self.w[name + ".weight"], self.w.get(name + ".bias"), rs, *[x for x, _ in segs])


def _pool(x, wgt):
  """fused_mean_variance over views: x [P,V,C], wgt [P,V] -> [P, 2C]."""
  mean = (x * wgt[..., None]).sum(1, keepdim=True)
  var = (wgt[..., None] * (x - mean) ** 2).sum(1)
  return torch.cat([mean[:, 0], var], -1)


def _attention(Q, K, Vv, valid, R, S, plant=None):
  """Ray-transformer attention (oracle ray_attention without its projections): query rows with valid == 0
  attend uniformly (mlp_network.py:23-24)."""
  sh = lambda t: t.view(R, S, 4, 32).transpose(1, 2)
  att = (sh(Q) / math.sqrt(32.0)) @ sh(K).transpose(2, 3)
  att = att.masked_fill(valid.view(R, 1, S, 1) == 0, -1e9)
  if plant == "keys_first256":
    att[..., 256:] = -math.inf
  return (torch.softmax(att, -1) @ sh(Vv)).transpose(1, 2).reshape(R * S, 128)


def _trunk(n, mv, C, feat, w1, mask, P, V, R, S, posenc):
  """run_trunk + run_point_tail (nets_f32.cu:600-658): -> G3 [P,128], X2 [M,128], masked vis2 [M], nvalid [P]."""
  M = P * V
  H1 = n.lin("base_fc.0", [(mv, V), (feat, 1)], "elu", P=P)
  X = n.lin("base_fc.2", [(H1, 1)], "elu", P=P)
  H2 = n.lin("vis_fc.0", [(X, 1)], "elu", rs=w1.reshape(M), P=P)
  XV = n.lin("vis_fc.2", [(H2, 1)], "elu", P=P)
  m = mask.reshape(M)
  vis1 = torch.sigmoid(XV[:, 128]) * m
  X2 = X + XV[:, :128]
  H3 = n.lin("vis_fc2.0", [(X2, 1)], "elu", rs=vis1, P=P)
  vis2 = n.lin("vis_fc2.2", [(H3, 1)], "sigmoid", P=P)[:, 0] * m
  vp, Xp = vis2.view(P, V), X2.view(P, V, 128)
  if n.plant == "pool2_first16":
    vp, Xp = vp[:, :16], Xp[:, :16]
  w2 = vp / (vp.sum(1, keepdim=True) + 1e-8)
  G = torch.cat([_pool(Xp, w2), w2.mean(1, keepdim=True)], -1)  # [P,257]
  GH = n.lin("geometry_fc.0", [(G, 1)], "elu")
  G2 = n.lin("geometry_fc.2", [(GH, 1)], "elu")
  if posenc:
    G2 = G2 + O.sinusoid_table(S).to(G2.device, G2.dtype).repeat(R, 1)
  nvalid = mask.view(P, V).sum(1)
  Q = n.lin("ray_attention.w_qs", [(G2, 1)], "none", acc_in=True)
  K = n.lin("ray_attention.w_ks", [(G2, 1)], "none", acc_in=True)
  Vv = n.lin("ray_attention.w_vs", [(G2, 1)], "none", acc_in=True)
  Oa = _attention(Q, K, Vv, (nvalid > 1).to(G2.dtype), R, S, n.plant)
  O2 = n.lin("ray_attention.fc", [(Oa, 1)], "none")
  G3 = F.layer_norm(O2 + G2, (128,), n.w["ray_attention.layer_norm.weight"], n.w["ray_attention.layer_norm.bias"],
                    eps=1e-6)
  return G3, X2, vis2, nvalid


def net_dynamic(w, pts, rgb_feat, ray_dir, mask, t, shift=0.0, mode="kernel", plant=None):
  """net_dynamic_f32 (train = true): pts [R,S,3], rgb_feat [R,S,V,35], ray_dir [R,3], mask [R,S,V,1] (float64),
  t (float) -> raw [R,S,4].  `w`: float64 parameters by state_dict name."""
  n = _Net(w, "dynamic", mode, plant)
  R, S, V, _ = rgb_feat.shape
  P, M = R * S, R * S * V
  dev = rgb_feat.device
  t_pe = O.periodic_embed(torch.tensor([[float(t)]], dtype=rgb_feat.dtype, device=dev), 10)
  # dyn_time_feat_kernel: fp32 SIMT in both precisions
  dfeat = F.elu(F.linear(F.elu(F.linear(t_pe, w["ray_dir_fc.0.weight"], w["ray_dir_fc.0.bias"])),
                         w["ray_dir_fc.2.weight"], w["ray_dir_fc.2.bias"]))
  feat = rgb_feat.reshape(M, 35) + dfeat
  mk = mask.reshape(P, V)
  w1 = mk / (mk.sum(1, keepdim=True) + 1e-8)
  mv = _pool(feat.view(P, V, 35), w1)
  G3, _, _, nvalid = _trunk(n, mv, 35, feat, w1, mk, P, V, R, S, True)
  ptspe = O.periodic_embed(pts.reshape(P, 3), 5)
  G4h = n.lin("ref_pts_fc.0", [(G3, 1), (ptspe, 1)], "elu")
  G4 = n.lin("ref_pts_fc.2", [(G4h, 1)], "elu")
  sh = n.lin("out_geometry_fc.0", [(G4, 1)], "elu", acc_in=True)
  sig = n.lin("out_geometry_fc.2", [(sh, 1)], "none")[:, 0] - shift
  dirpe = O.periodic_embed(ray_dir, 4)
  ch = n.lin("rgb_fc.0", [(G4, 1), (dirpe, S)], "elu")
  ch2 = n.lin("rgb_fc.2", [(ch, 1)], "elu")
  rgb = n.lin("rgb_fc.4", [(ch2, 1)], "sigmoid")
  rgb = rgb.masked_fill((nvalid < 1)[:, None], 0.0)
  sig = sig.masked_fill(nvalid < 1, -1e9)
  return torch.cat([rgb, sig[:, None]], -1).view(R, S, 4)


def net_static(w, pts, ref_rays, src_rays, rgb_feat, ray_diff, mask, anti_alias=True, mask_rgb=False, mode="kernel",
               plant=None):
  """net_static_f32 (train = true); shapes as oracle.net_static, all float64 -> raw [R,S,4]."""
  n = _Net(w, "static", mode, plant)
  R, S, V, _ = rgb_feat.shape
  P, M = R * S, R * S * V
  ptspe = O.periodic_embed(pts.reshape(P, 3), 5)
  srcpe = O.periodic_embed(src_rays.reshape(M, 6), 5)
  refpe = O.periodic_embed(ref_rays, 5)
  rd = ray_diff.reshape(M, 4)
  H0 = n.lin("ray_dir_fc.0", [(ptspe, V), (srcpe, 1), (rd, 1)], "elu", P=P)
  SF = n.lin("ray_dir_fc.2", [(H0, 1)], "none", P=P)
  reff = n.lin("ref_feature_fc.0", [(refpe, 1)], "none")
  rf = rgb_feat.reshape(M, 35)
  mk = mask.reshape(P, V)
  if mask_rgb:
    mk = mk * (rf[:, :3].sum(-1) > 1e-3).to(mk.dtype).view(P, V)
  feat70 = torch.cat([rf, SF * reff.repeat_interleave(S * V, 0)], -1)
  if anti_alias:
    e = torch.exp(torch.abs(w["s"]) * (rd[:, 3].view(P, V) - 1))
    w1 = (e - e.min(1, keepdim=True)[0]) * mk
    w1 = w1 / (w1.sum(1, keepdim=True) + 1e-8)
  else:
    w1 = mk / (mk.sum(1, keepdim=True) + 1e-8)
  mv = _pool(feat70.view(P, V, 70), w1)
  G3, X2, vis2, nvalid = _trunk(n, mv, 70, feat70, w1, mk, P, V, R, S, False)
  sh = n.lin("out_geometry_fc.0", [(G3, 1)], "elu", acc_in=True)
  sig = n.lin("out_geometry_fc.2", [(sh, 1)], "none")[:, 0]
  ch = n.lin("rgb_fc.0", [(G3, V), (X2, 1), (vis2[:, None], 1), (rd, 1)], "elu", P=P)
  ch2 = n.lin("rgb_fc.2", [(ch, 1)], "elu", P=P)
  logit = n.lin("rgb_fc.4", [(ch2, 1)], "none", P=P)[:, 0].view(P, V)
  blend = torch.softmax(logit.masked_fill(mk == 0, -1e9), 1)
  rgb = (blend[..., None] * rf[:, :3].view(P, V, 3)).sum(1)
  if plant == "blend_first16":
    b16 = torch.softmax(logit.masked_fill(mk == 0, -1e9)[:, :16], 1)
    rgb = (b16[..., None] * rf[:, :3].view(P, V, 3)[:, :16]).sum(1)
  sig = sig.masked_fill(nvalid < 1, -1e9)
  return torch.cat([rgb, sig[:, None]], -1).view(R, S, 4)


def motion_mlp(w, xyzt, mode="kernel", plant=None, stats=None):
  """motion_train_forward: xyzt [N,4] float64 -> coeff [N, 3 num_basis].  `stats`, a dict, receives per ReLU layer
  (pre-activations near 0, all pre-activations)."""
  n = _Net(w, "motion", mode, plant, stats)
  x0 = O.periodic_embed(xyzt, 16, linspace=True)
  h = x0
  for i in range(8):
    h = n.lin("pts_linears.%d" % i, [(x0, 1), (h, 1)] if i == 5 else [(h, 1)], "relu")
  return n.lin("coeff_linear", [(h, 1)], "none")


# ---------------------------------------------------------------------------------------------------------------
# Cases and comparison, shared by the CPU and GPU tests
# ---------------------------------------------------------------------------------------------------------------
def make_net_case(kind, R, S, V, aa=False, mrgb=False, seed=0):
  """Seeded module and inputs (CPU, fp32) of one net case, and its upstream gradient (zero where sigma is -1e9).
  Masks include a point no view sees and a point with exactly one valid view (a masked query row); ray_diff has
  cos in [0.7, 1] so that d s is well conditioned."""
  from dynibar_b200 import mlp_network as nets, synthetic
  torch.manual_seed(seed)
  args = synthetic.make_args(int(aa), int(mrgb))
  if kind == "dynamic":
    mod = nets.DynibarDynamic(args, 32, S, shift=5.0)
    with torch.no_grad():
      mod.out_geometry_fc[2].bias.fill_(1.0)
  else:
    mod = nets.DynibarStatic(args, 32, S)
    with torch.no_grad():
      mod.out_geometry_fc[2].bias.fill_(0.5)
  g = torch.Generator().manual_seed(seed + 1)
  c = dict(kind=kind, aa=aa, mrgb=mrgb, mod=mod)
  c["pts"] = torch.randn(R, S, 3, generator=g) * 2
  feat = torch.randn(R, S, V, 35, generator=g)
  feat[..., :3] = torch.rand(R, S, V, 3, generator=g)
  mask = (torch.rand(R, S, V, 1, generator=g) > 0.3).float()
  mask[0, 0] = 0.0
  mask[0, 1] = 0.0
  mask[0, 1, 0] = 1.0
  if V > 1:
    mask[0, 2] = 1.0  # every view valid
  if mrgb:
    feat[0, 3, 0, :3] = 0.0  # a dark source colour: masked out by mask_rgb
  c["feat"], c["mask"] = feat, mask
  c["ray_dir"] = F.normalize(torch.randn(R, 3, generator=g), dim=-1)
  c["t"] = float(torch.tensor(0.4, dtype=torch.float32))  # the library embeds the time from an fp32 value
  c["ref_rays"] = torch.randn(R, 6, generator=g)
  c["src_rays"] = torch.randn(R, S, V, 6, generator=g)
  c["ray_diff"] = torch.cat([F.normalize(torch.randn(R, S, V, 3, generator=g), dim=-1),
                             torch.rand(R, S, V, 1, generator=g) * 0.3 + 0.7], -1)
  meff = mask
  if kind == "static" and mrgb:
    meff = mask * (feat[..., :3].sum(-1, keepdim=True) > 1e-3).float()
  if kind == "static" and aa:
    _condition_aa(c["ray_diff"], mask, meff)
  live = (meff.sum(2) >= 1).float()
  c["gen"] = torch.randn(R, S, 4, generator=g) * torch.cat([live.expand(-1, -1, 3), live], -1)
  return c


def _condition_aa(ray_diff, mask, meff):
  """In place: no point keeps exactly one view of nonzero anti-aliased pooling weight u_v = (e_v - min e) m_v.
  There w = u / (u + 1e-8) is 1 to within 1e-8 / u, so its derivative, and with it d s, is a difference of nearly
  equal fp32 numbers that carries no significant bit.  A point with one valid view gets that view's cos swapped
  with the minimum (u = 0: no weight, no gradient); a point with more gets a second nonzero-weight view."""
  V = mask.shape[2]
  cos, m, me = ray_diff[..., 3].view(-1, V), mask.view(-1, V), meff.view(-1, V)
  am = cos.argmin(1)
  nz = me.clone()
  nz[torch.arange(nz.shape[0]), am] = 0.0
  for p in torch.nonzero(nz.sum(1) == 1).flatten().tolist():
    v = int(torch.nonzero(nz[p])[0])
    if me[p].sum() == 1:
      cos[p, v], cos[p, am[p]] = cos[p, am[p]].clone(), cos[p, v].clone()
    else:  # add a valid view that mask_rgb keeps (m == me there unless the colour is dark)
      free = torch.nonzero((m[p] == 0) & (torch.arange(V) != am[p])).flatten()
      m[p, free[0]] = 1.0
      me[p, free[0]] = 1.0


def make_motion_case(N, num_basis, seed=0):
  from dynibar_b200 import mlp_network as nets
  torch.manual_seed(seed)
  mod = nets.MotionMLP(num_basis=num_basis)
  with torch.no_grad():  # coeff_linear starts at zero (mlp_network.py:602-603): give it a gradient path
    mod.coeff_linear.weight.normal_(0.0, 0.05)
    mod.coeff_linear.bias.normal_(0.0, 0.05)
  g = torch.Generator().manual_seed(seed + 1)
  xyzt = torch.cat([torch.randn(N, 3, generator=g), torch.rand(N, 1, generator=g)], -1)
  return dict(kind="motion", mod=mod, xyzt=xyzt, gen=torch.randn(N, 3 * num_basis, generator=g))


def reference(c, device, mode="kernel", plant=None, stats=None, dtype=torch.float64):
  """Forward and every gradient of case `c` on `device`: {"out": raw / coeff, "<param>": d param,
  "rgb_feat" / "pts" / "xyzt": d input}.  dtype=torch.float32 evaluates the same arithmetic in float32, which
  estimates how far the library's own fp32 arithmetic can drift from the float64 evaluation."""
  d = lambda x: x.detach().to(device, dtype, copy=True)  # never the case's own tensors
  w = {k: d(p.detach()).requires_grad_(True) for k, p in c["mod"].named_parameters()}
  if c["kind"] == "motion":
    x = d(c["xyzt"]).requires_grad_(True)
    out = motion_mlp(w, x, mode, plant, stats)
    ins = {"xyzt": x}
  elif c["kind"] == "dynamic":
    pts, feat = d(c["pts"]).requires_grad_(True), d(c["feat"]).requires_grad_(True)
    out = net_dynamic(w, pts, feat, d(c["ray_dir"]), d(c["mask"]), c["t"], float(c["mod"].shift), mode, plant)
    ins = {"pts": pts, "rgb_feat": feat}
  else:
    feat = d(c["feat"]).requires_grad_(True)
    out = net_static(w, d(c["pts"]), d(c["ref_rays"]), d(c["src_rays"]), feat, d(c["ray_diff"]), d(c["mask"]),
                     c["aa"], c["mrgb"], mode, plant)
    ins = {"rgb_feat": feat}
  (out * d(c["gen"])).sum().backward()
  res = {"out": out.detach()}
  res.update({k: v.grad for k, v in w.items()})
  res.update({k: v.grad for k, v in ins.items()})
  return res


# Cases of the GPU test: net cases (R, S, V, anti_alias, mask_rgb; the last two apply to the static net) and
# MotionMLP cases (N, num_basis).
NET_CASES = {
    "all_simt": (6, 16, 5, True, False),
    "fwd_tc_only": (40, 16, 3, True, False),
    "view_tc": (40, 16, 8, False, False),
    "ragged": (131, 16, 11, True, False),
    "per_ray_tc": (2053, 4, 2, False, False),
    "v1": (128, 32, 1, False, True),
    "v16": (64, 32, 16, True, False),
    "bench_like": (256, 64, 8, True, True),
}
MOTION_CASES = {
    "n1": (1, 6),
    "n127": (127, 6),
    "n128": (128, 4),
    "n2047": (2047, 8),
    "n2048": (2048, 4),
    "n2049": (2049, 6),
    "n65573_nb4": (65573, 4),
    "n65573_nb8": (65573, 8),
}

# Bars of the GPU comparison: per (net, precision) and compared tensor, (relative L2 error, max |error| /
# max |reference|).  Tensors not listed take DEFAULT_BAR.  How they were set is in tests/test_train_stage_gpu.py.
DEFAULT_BAR = {"bf16": (1e-3, 1e-2), "fp32": (1e-4, 1e-3)}
BARS = {
    ("dynamic", "bf16"): {
        "base_fc.0.bias": (9e-03, 1e-02),  # 4.40e-03 4.79e-03 v16
        "base_fc.0.weight": (1e-02, 2e-02),  # 4.66e-03 5.36e-03 v16
        "base_fc.2.bias": (1e-02, 2e-02),  # 4.68e-03 5.09e-03 v16
        "base_fc.2.weight": (9e-03, 2e-02),  # 4.44e-03 5.56e-03 v16
        "geometry_fc.0.bias": (7e-03, 6e-03),  # 3.40e-03 2.90e-03 v16
        "geometry_fc.0.weight": (9e-03, 8e-03),  # 4.10e-03 3.89e-03 v16
        "geometry_fc.2.bias": (5e-03, 5e-03),  # 2.21e-03 2.01e-03 v16
        "geometry_fc.2.weight": (7e-03, 8e-03),  # 3.26e-03 3.51e-03 v16
        "out": (1e-04, 6e-04),  # 3.51e-05 2.68e-04 bench_like
        "out_geometry_fc.0.bias": (7e-04, 1e-03),  # 3.18e-04 4.91e-04 fwd_tc_only
        "out_geometry_fc.0.weight": (5e-03, 5e-03),  # 2.07e-03 2.36e-03 v16
        "out_geometry_fc.2.bias": (1e-04, 1e-04),  # 1.03e-06 1.03e-06 v16
        "out_geometry_fc.2.weight": (5e-03, 7e-03),  # 2.45e-03 3.23e-03 v16
        "pts": (4e-03, 7e-03),  # 1.88e-03 3.07e-03 v16
        "ray_attention.fc.weight": (6e-03, 6e-03),  # 2.80e-03 2.98e-03 v16
        "ray_attention.layer_norm.bias": (5e-03, 5e-03),  # 2.05e-03 2.29e-03 v16
        "ray_attention.layer_norm.weight": (4e-03, 3e-03),  # 1.52e-03 1.39e-03 ragged
        "ray_attention.w_ks.weight": (9e-03, 7e-03),  # 4.27e-03 3.32e-03 ragged
        "ray_attention.w_qs.weight": (8e-03, 9e-03),  # 3.60e-03 4.28e-03 ragged
        "ray_attention.w_vs.weight": (6e-03, 6e-03),  # 2.82e-03 2.58e-03 v16
        "ray_dir_fc.0.bias": (8e-03, 2e-02),  # 3.86e-03 5.07e-03 v16
        "ray_dir_fc.0.weight": (8e-03, 2e-02),  # 3.86e-03 5.07e-03 v16
        "ray_dir_fc.2.bias": (8e-03, 7e-03),  # 3.88e-03 3.11e-03 v16
        "ray_dir_fc.2.weight": (8e-03, 7e-03),  # 3.88e-03 3.11e-03 v16
        "ref_pts_fc.0.bias": (3e-03, 2e-03),  # 1.16e-03 9.36e-04 v16
        "ref_pts_fc.0.weight": (4e-03, 3e-03),  # 1.89e-03 1.36e-03 v16
        "ref_pts_fc.2.bias": (1e-03, 2e-03),  # 4.66e-04 5.33e-04 v16
        "ref_pts_fc.2.weight": (4e-03, 7e-03),  # 1.67e-03 3.04e-03 v16
        "rgb_fc.0.bias": (2e-03, 2e-03),  # 6.88e-04 8.14e-04 bench_like
        "rgb_fc.0.weight": (3e-03, 2e-03),  # 1.21e-03 8.42e-04 bench_like
        "rgb_fc.2.bias": (5e-04, 7e-04),  # 2.14e-04 3.36e-04 fwd_tc_only
        "rgb_fc.2.weight": (4e-03, 5e-03),  # 1.76e-03 2.19e-03 bench_like
        "rgb_fc.4.bias": (1e-04, 1e-04),  # 6.73e-06 7.52e-06 v16
        "rgb_fc.4.weight": (5e-03, 4e-03),  # 2.33e-03 1.99e-03 bench_like
        "rgb_feat": (8e-03, 2e-02),  # 3.80e-03 5.61e-03 v16
        "vis_fc.0.bias": (1e-02, 2e-02),  # 4.77e-03 5.77e-03 v16
        "vis_fc.0.weight": (9e-03, 1e-02),  # 4.32e-03 4.87e-03 v16
        "vis_fc.2.bias": (1e-02, 2e-02),  # 4.77e-03 5.87e-03 v16
        "vis_fc.2.weight": (1e-02, 2e-02),  # 4.89e-03 6.47e-03 v16
        "vis_fc2.0.bias": (9e-03, 7e-03),  # 4.03e-03 3.43e-03 bench_like
        "vis_fc2.0.weight": (1e-02, 2e-02),  # 4.66e-03 5.69e-03 bench_like
        "vis_fc2.2.bias": (3e-04, 2e-03),  # 1.31e-04 5.35e-04 bench_like
        "vis_fc2.2.weight": (2e-02, 2e-02),  # 6.29e-03 5.52e-03 bench_like
    },
    ("dynamic", "fp32"): {
        "base_fc.0.bias": (1e-05, 1e-05),  # 1.27e-06 1.46e-06 v16
        "base_fc.0.weight": (1e-05, 1e-05),  # 1.37e-06 2.17e-06 v16
        "base_fc.2.bias": (1e-05, 1e-05),  # 1.32e-06 1.01e-06 fwd_tc_only
        "base_fc.2.weight": (1e-05, 1e-05),  # 1.83e-06 2.56e-06 v16
        "geometry_fc.0.bias": (1e-05, 1e-05),  # 1.28e-06 1.38e-06 fwd_tc_only
        "geometry_fc.0.weight": (1e-05, 1e-05),  # 1.23e-06 1.36e-06 v16
        "geometry_fc.2.bias": (1e-05, 1e-05),  # 1.11e-06 1.11e-06 fwd_tc_only
        "geometry_fc.2.weight": (1e-05, 1e-05),  # 1.70e-06 2.84e-06 v1
        "out": (1e-05, 1e-05),  # 3.94e-08 9.33e-08 all_simt
        "out_geometry_fc.0.bias": (1e-05, 1e-05),  # 6.75e-07 1.44e-06 v16
        "out_geometry_fc.0.weight": (1e-05, 1e-05),  # 1.07e-06 2.16e-06 bench_like
        "out_geometry_fc.2.bias": (1e-05, 1e-05),  # 1.03e-06 1.03e-06 v16
        "out_geometry_fc.2.weight": (1e-05, 1e-05),  # 1.00e-06 1.68e-06 bench_like
        "pts": (1e-05, 1e-05),  # 6.31e-07 8.28e-07 per_ray_tc
        "ray_attention.fc.weight": (1e-05, 1e-05),  # 1.11e-06 1.76e-06 fwd_tc_only
        "ray_attention.layer_norm.bias": (1e-05, 1e-05),  # 1.02e-06 1.25e-06 fwd_tc_only
        "ray_attention.layer_norm.weight": (1e-05, 1e-05),  # 6.45e-07 5.89e-07 fwd_tc_only
        "ray_attention.w_ks.weight": (1e-05, 1e-05),  # 2.43e-06 2.70e-06 fwd_tc_only
        "ray_attention.w_qs.weight": (1e-05, 1e-05),  # 2.54e-06 2.17e-06 fwd_tc_only
        "ray_attention.w_vs.weight": (1e-05, 1e-05),  # 1.10e-06 2.18e-06 fwd_tc_only
        "ray_dir_fc.0.bias": (1e-05, 1e-05),  # 1.19e-06 1.23e-06 v16
        "ray_dir_fc.0.weight": (1e-05, 1e-05),  # 1.19e-06 1.22e-06 v16
        "ray_dir_fc.2.bias": (1e-05, 1e-05),  # 1.21e-06 1.08e-06 v16
        "ray_dir_fc.2.weight": (1e-05, 1e-05),  # 1.22e-06 1.16e-06 v16
        "ref_pts_fc.0.bias": (1e-05, 1e-05),  # 8.28e-07 9.40e-07 v16
        "ref_pts_fc.0.weight": (1e-05, 1e-05),  # 9.75e-07 2.03e-06 bench_like
        "ref_pts_fc.2.bias": (1e-05, 1e-05),  # 6.89e-07 7.34e-07 fwd_tc_only
        "ref_pts_fc.2.weight": (1e-05, 1e-05),  # 1.04e-06 2.11e-06 bench_like
        "rgb_fc.0.bias": (1e-05, 1e-05),  # 5.94e-07 7.39e-07 bench_like
        "rgb_fc.0.weight": (1e-05, 1e-05),  # 8.80e-07 2.03e-06 bench_like
        "rgb_fc.2.bias": (1e-05, 1e-05),  # 4.32e-07 7.30e-07 v1
        "rgb_fc.2.weight": (1e-05, 1e-05),  # 1.22e-06 2.03e-06 bench_like
        "rgb_fc.4.bias": (1e-05, 1e-05),  # 7.25e-07 5.85e-07 bench_like
        "rgb_fc.4.weight": (1e-05, 1e-05),  # 1.37e-06 1.51e-06 bench_like
        "rgb_feat": (1e-05, 1e-05),  # 7.01e-07 9.38e-07 v16
        "vis_fc.0.bias": (1e-05, 1e-05),  # 1.33e-06 1.86e-06 fwd_tc_only
        "vis_fc.0.weight": (1e-05, 1e-05),  # 1.87e-06 3.03e-06 v16
        "vis_fc.2.bias": (1e-05, 1e-05),  # 1.43e-06 1.18e-06 fwd_tc_only
        "vis_fc.2.weight": (1e-05, 1e-05),  # 2.17e-06 3.19e-06 v16
        "vis_fc2.0.bias": (3e-05, 3e-05),  # 1.08e-05 1.33e-05 per_ray_tc
        "vis_fc2.0.weight": (1e-05, 1e-05),  # 1.55e-06 1.92e-06 bench_like
        "vis_fc2.2.bias": (1e-05, 1e-05),  # 1.14e-06 4.22e-06 ragged
        "vis_fc2.2.weight": (1e-05, 1e-05),  # 1.68e-06 1.95e-06 per_ray_tc
    },
    ("motion", "bf16"): {
        "coeff_linear.bias": (1e-04, 1e-04),  # 4.51e-07 5.85e-07 n65573_nb4
        "coeff_linear.weight": (1e-03, 2e-03),  # 4.62e-04 6.05e-04 n2049
        "out": (3e-04, 4e-03),  # 1.46e-04 1.80e-03 n65573_nb8
        "pts_linears.0.bias": (2e-02, 3e-02),  # 9.36e-03 1.02e-02 n65573_nb8
        "pts_linears.0.weight": (2e-02, 3e-02),  # 9.12e-03 1.05e-02 n65573_nb8
        "pts_linears.1.bias": (3e-02, 5e-02),  # 1.03e-02 2.28e-02 n65573_nb8
        "pts_linears.1.weight": (2e-02, 2e-01),  # 9.52e-03 5.10e-02 n65573_nb8
        "pts_linears.2.bias": (2e-02, 6e-02),  # 9.31e-03 2.61e-02 n65573_nb8
        "pts_linears.2.weight": (2e-02, 7e-02),  # 9.14e-03 3.21e-02 n65573_nb8
        "pts_linears.3.bias": (2e-02, 4e-02),  # 8.51e-03 1.52e-02 n65573_nb4
        "pts_linears.3.weight": (2e-02, 5e-02),  # 8.26e-03 2.36e-02 n65573_nb4
        "pts_linears.4.bias": (2e-02, 4e-02),  # 7.65e-03 1.54e-02 n2047
        "pts_linears.4.weight": (2e-02, 4e-02),  # 7.32e-03 1.94e-02 n2047
        "pts_linears.5.bias": (2e-02, 2e-02),  # 6.91e-03 9.65e-03 n2047
        "pts_linears.5.weight": (2e-02, 4e-02),  # 6.41e-03 1.64e-02 n2047
        "pts_linears.6.bias": (2e-02, 4e-02),  # 7.92e-03 1.91e-02 n2047
        "pts_linears.6.weight": (2e-02, 7e-02),  # 7.19e-03 3.28e-02 n2047
        "pts_linears.7.bias": (2e-02, 8e-02),  # 8.49e-03 3.54e-02 n2047
        "pts_linears.7.weight": (2e-02, 9e-02),  # 7.90e-03 4.41e-02 n2047
        "xyzt": (2e-02, 2e-01),  # 6.54e-03 7.14e-02 n2047
    },
    ("motion", "fp32"): {
        "coeff_linear.bias": (1e-05, 1e-05),  # 4.45e-07 5.85e-07 n65573_nb4
        "coeff_linear.weight": (1e-05, 1e-05),  # 1.27e-06 1.81e-06 n65573_nb8
        "out": (1e-05, 1e-05),  # 3.41e-07 7.07e-07 n65573_nb8
        "pts_linears.0.bias": (1e-02, 5e-02),  # 4.86e-03 2.48e-02 n2049
        "pts_linears.0.weight": (1e-02, 7e-02),  # 4.50e-03 3.27e-02 n2049
        "pts_linears.1.bias": (5e-03, 7e-03),  # 2.16e-03 3.08e-03 n2049
        "pts_linears.1.weight": (5e-03, 2e-02),  # 2.20e-03 5.99e-03 n2049
        "pts_linears.2.bias": (5e-03, 3e-02),  # 2.12e-03 1.11e-02 n2049
        "pts_linears.2.weight": (5e-03, 3e-02),  # 2.14e-03 1.24e-02 n2049
        "pts_linears.3.bias": (2e-03, 2e-03),  # 9.41e-04 9.26e-04 n65573_nb4
        "pts_linears.3.weight": (3e-03, 3e-03),  # 1.00e-03 1.06e-03 n65573_nb4
        "pts_linears.4.bias": (2e-03, 5e-03),  # 8.27e-04 2.09e-03 n65573_nb4
        "pts_linears.4.weight": (2e-03, 6e-03),  # 8.82e-04 2.56e-03 n65573_nb4
        "pts_linears.5.bias": (2e-03, 6e-03),  # 9.18e-04 2.99e-03 n65573_nb4
        "pts_linears.5.weight": (2e-03, 7e-03),  # 9.11e-04 3.46e-03 n65573_nb4
        "pts_linears.6.bias": (2e-03, 6e-03),  # 6.67e-04 2.66e-03 n65573_nb4
        "pts_linears.6.weight": (2e-03, 9e-03),  # 6.72e-04 4.46e-03 n65573_nb4
        "pts_linears.7.bias": (9e-04, 3e-03),  # 4.03e-04 1.33e-03 n65573_nb4
        "pts_linears.7.weight": (9e-04, 4e-03),  # 4.05e-04 1.97e-03 n65573_nb4
        "xyzt": (2e-03, 8e-02),  # 9.01e-04 3.97e-02 n65573_nb4
    },
    ("static", "bf16"): {
        "base_fc.0.bias": (8e-03, 2e-02),  # 3.85e-03 5.00e-03 v16
        "base_fc.0.weight": (9e-03, 8e-03),  # 4.21e-03 3.90e-03 v16
        "base_fc.2.bias": (8e-03, 9e-03),  # 3.63e-03 4.21e-03 v16
        "base_fc.2.weight": (7e-03, 1e-02),  # 3.08e-03 4.56e-03 v16
        "geometry_fc.0.bias": (4e-03, 4e-03),  # 1.60e-03 1.52e-03 v16
        "geometry_fc.0.weight": (6e-03, 1e-02),  # 2.91e-03 4.88e-03 v16
        "geometry_fc.2.bias": (2e-03, 3e-03),  # 8.78e-04 1.20e-03 v16
        "geometry_fc.2.weight": (4e-03, 6e-03),  # 1.69e-03 2.91e-03 v16
        "out": (7e-04, 5e-03),  # 3.02e-04 2.12e-03 fwd_tc_only
        "out_geometry_fc.0.bias": (2e-03, 3e-03),  # 7.28e-04 1.26e-03 v16
        "out_geometry_fc.0.weight": (5e-03, 8e-03),  # 2.34e-03 3.95e-03 v16
        "out_geometry_fc.2.bias": (1e-04, 1e-04),  # 1.03e-06 1.03e-06 v16
        "out_geometry_fc.2.weight": (7e-03, 8e-03),  # 3.16e-03 3.97e-03 v16
        "ray_attention.fc.weight": (4e-03, 5e-03),  # 1.99e-03 2.33e-03 v16
        "ray_attention.layer_norm.bias": (2e-03, 2e-03),  # 7.77e-04 8.02e-04 v16
        "ray_attention.layer_norm.weight": (3e-03, 3e-03),  # 1.29e-03 1.21e-03 fwd_tc_only
        "ray_attention.w_ks.weight": (2e-02, 2e-02),  # 6.32e-03 8.46e-03 v16
        "ray_attention.w_qs.weight": (9e-03, 9e-03),  # 4.12e-03 4.28e-03 v16
        "ray_attention.w_vs.weight": (5e-03, 6e-03),  # 2.37e-03 2.64e-03 v16
        "ray_dir_fc.0.bias": (7e-03, 8e-03),  # 3.16e-03 3.86e-03 ragged
        "ray_dir_fc.0.weight": (8e-03, 8e-03),  # 3.51e-03 3.77e-03 ragged
        "ray_dir_fc.2.bias": (6e-03, 7e-03),  # 2.96e-03 3.08e-03 v16
        "ray_dir_fc.2.weight": (7e-03, 5e-03),  # 3.02e-03 2.17e-03 v1
        "ref_feature_fc.0.bias": (2e-02, 2e-02),  # 7.86e-03 9.33e-03 v16
        "ref_feature_fc.0.weight": (7e-03, 5e-03),  # 3.21e-03 2.19e-03 v16
        "rgb_fc.0.bias": (2e-03, 8e-03),  # 9.59e-04 3.74e-03 bench_like
        "rgb_fc.0.weight": (3e-02, 2e-02),  # 1.12e-02 8.17e-03 bench_like
        "rgb_fc.2.bias": (1e-03, 1e-02),  # 4.84e-04 4.92e-03 v16
        "rgb_fc.2.weight": (4e-02, 6e-02),  # 1.76e-02 2.59e-02 v16
        "rgb_fc.4.bias": (1e-04, 1e-04),  # 3.85e-06 1.51e-05 bench_like
        "rgb_fc.4.weight": (6e-02, 8e-02),  # 2.53e-02 4.00e-02 bench_like
        "rgb_feat": (2e-03, 3e-03),  # 6.73e-04 1.00e-03 ragged
        "s": (2e-02, 2e-02),  # 6.22e-03 6.22e-03 bench_like
        "vis_fc.0.bias": (8e-03, 2e-02),  # 3.87e-03 5.36e-03 v16
        "vis_fc.0.weight": (7e-03, 8e-03),  # 3.40e-03 3.72e-03 v16
        "vis_fc.2.bias": (8e-03, 9e-03),  # 3.59e-03 4.11e-03 v16
        "vis_fc.2.weight": (8e-03, 1e-02),  # 3.66e-03 4.50e-03 v16
        "vis_fc2.0.bias": (5e-03, 5e-03),  # 2.18e-03 2.20e-03 v16
        "vis_fc2.0.weight": (9e-03, 2e-02),  # 4.31e-03 5.62e-03 ragged
        "vis_fc2.2.bias": (2e-04, 7e-04),  # 6.76e-05 3.18e-04 view_tc
        "vis_fc2.2.weight": (2e-02, 2e-02),  # 6.00e-03 6.27e-03 ragged
    },
    ("static", "fp32"): {
        "base_fc.0.bias": (1e-05, 1e-05),  # 1.67e-06 1.84e-06 fwd_tc_only
        "base_fc.0.weight": (1e-05, 1e-05),  # 3.39e-06 4.50e-06 fwd_tc_only
        "base_fc.2.bias": (1e-05, 1e-05),  # 1.55e-06 1.74e-06 fwd_tc_only
        "base_fc.2.weight": (1e-05, 1e-05),  # 3.39e-06 3.06e-06 fwd_tc_only
        "geometry_fc.0.bias": (1e-05, 1e-05),  # 1.40e-06 1.74e-06 fwd_tc_only
        "geometry_fc.0.weight": (1e-05, 1e-05),  # 3.33e-06 3.45e-06 fwd_tc_only
        "geometry_fc.2.bias": (1e-05, 1e-05),  # 1.39e-06 1.50e-06 fwd_tc_only
        "geometry_fc.2.weight": (1e-05, 1e-05),  # 3.21e-06 3.03e-06 fwd_tc_only
        "out": (1e-05, 2e-05),  # 4.15e-07 6.58e-06 fwd_tc_only
        "out_geometry_fc.0.bias": (1e-05, 1e-05),  # 1.26e-06 1.96e-06 fwd_tc_only
        "out_geometry_fc.0.weight": (1e-05, 1e-05),  # 3.01e-06 2.84e-06 fwd_tc_only
        "out_geometry_fc.2.bias": (1e-05, 1e-05),  # 1.03e-06 1.03e-06 v16
        "out_geometry_fc.2.weight": (1e-05, 1e-05),  # 2.98e-06 2.29e-06 fwd_tc_only
        "ray_attention.fc.weight": (1e-05, 1e-05),  # 1.62e-06 2.23e-06 fwd_tc_only
        "ray_attention.layer_norm.bias": (1e-05, 1e-05),  # 1.35e-06 1.47e-06 fwd_tc_only
        "ray_attention.layer_norm.weight": (1e-05, 2e-05),  # 3.53e-06 5.16e-06 fwd_tc_only
        "ray_attention.w_ks.weight": (1e-05, 1e-05),  # 4.10e-06 4.98e-06 ragged
        "ray_attention.w_qs.weight": (1e-05, 1e-05),  # 3.95e-06 4.77e-06 ragged
        "ray_attention.w_vs.weight": (1e-05, 1e-05),  # 1.94e-06 3.32e-06 fwd_tc_only
        "ray_dir_fc.0.bias": (1e-05, 1e-05),  # 1.12e-06 1.23e-06 fwd_tc_only
        "ray_dir_fc.0.weight": (1e-05, 1e-05),  # 1.39e-06 1.68e-06 fwd_tc_only
        "ray_dir_fc.2.bias": (1e-05, 1e-05),  # 1.10e-06 1.13e-06 fwd_tc_only
        "ray_dir_fc.2.weight": (1e-05, 1e-05),  # 1.42e-06 1.68e-06 fwd_tc_only
        "ref_feature_fc.0.bias": (1e-05, 1e-05),  # 1.62e-06 2.22e-06 v16
        "ref_feature_fc.0.weight": (1e-05, 1e-05),  # 1.34e-06 1.13e-06 fwd_tc_only
        "rgb_fc.0.bias": (1e-05, 1e-05),  # 3.19e-07 1.91e-06 ragged
        "rgb_fc.0.weight": (1e-05, 1e-05),  # 3.49e-06 2.89e-06 ragged
        "rgb_fc.2.bias": (1e-05, 2e-05),  # 9.80e-07 5.38e-06 ragged
        "rgb_fc.2.weight": (1e-05, 2e-05),  # 3.63e-06 5.71e-06 ragged
        "rgb_fc.4.bias": (1e-05, 3e-05),  # 3.51e-06 1.19e-05 v16
        "rgb_fc.4.weight": (1e-05, 2e-05),  # 4.31e-06 5.63e-06 ragged
        "rgb_feat": (1e-05, 1e-05),  # 3.95e-07 1.94e-06 ragged
        "s": (2e-02, 2e-02),  # 5.28e-03 5.28e-03 fwd_tc_only
        "vis_fc.0.bias": (1e-05, 1e-05),  # 1.82e-06 2.12e-06 fwd_tc_only
        "vis_fc.0.weight": (1e-05, 1e-05),  # 3.63e-06 4.01e-06 fwd_tc_only
        "vis_fc.2.bias": (1e-05, 1e-05),  # 1.58e-06 1.61e-06 fwd_tc_only
        "vis_fc.2.weight": (1e-05, 1e-05),  # 2.52e-06 3.44e-06 fwd_tc_only
        "vis_fc2.0.bias": (4e-05, 5e-05),  # 1.63e-05 2.00e-05 fwd_tc_only
        "vis_fc2.0.weight": (1e-05, 1e-05),  # 2.00e-06 2.59e-06 fwd_tc_only
        "vis_fc2.2.bias": (1e-05, 2e-05),  # 1.17e-06 5.47e-06 view_tc
        "vis_fc2.2.weight": (1e-05, 1e-05),  # 1.97e-06 2.35e-06 fwd_tc_only
    },
}


def bar(kind, prec, name):
  return BARS.get((kind, prec), {}).get(name, DEFAULT_BAR[prec])


def companion(kind, name, V):
  """The tensor whose norm a gradient's error is measured against, when the gradient is a sum whose terms cancel,
  so that its own norm is far below the size of its terms and of their rounding: the blending head's biases
  (sum over the views of a point of d logit_v is 0, a softmax being invariant to a common shift; rgb_fc.4.bias is
  0 in exact arithmetic), vis_fc2.2's bias (a sum over views of the derivative of weights normalised to sum 1);
  at V = 1, all of vis_fc2 (w2 = vis2 / (vis2 + 1e-8) is 1 to within 1e-8 / vis2).  The companion is the weight
  gradient of the same layer, the same dZ times that layer's input."""
  if V == 1 and name.startswith("vis_fc2."):
    return "vis_fc.2.weight"
  if kind == "static" and name in ("rgb_fc.0.bias", "rgb_fc.2.bias", "rgb_fc.4.bias"):
    return name[:-4] + "weight"
  if name == "vis_fc2.2.bias":
    return "vis_fc2.2.weight"
  return None


def errors(kind, got, ref, V=None):
  """{name: (relative L2 error, max |error| / max |ref|)} over every tensor of `ref`; sigma entries that are -1e9
  in the reference must be exactly -1e9 and are left out of the norms."""
  out = {}
  for name, b in ref.items():
    b = b.double()
    a = got[name].detach().to(b.device, torch.float64).reshape(b.shape)
    if name == "out" and kind != "motion":
      masked = b == -1e9
      if not torch.equal(a[masked], b[masked]):
        out[name] = (float("inf"), float("inf"))
        continue
      a, b = a[~masked], b[~masked]
    e = a - b
    cn = companion(kind, name, V)
    scale = ref[cn].double() if cn else b
    nb, mb = float(scale.norm()), float(scale.abs().max())
    out[name] = (float(e.norm()) / nb if nb > 0 else float(e.norm()),
                 float(e.abs().max()) / mb if mb > 0 else float(e.abs().max()))
  return out


def ratios(kind, prec, got, ref, V=None):
  """Per tensor: the larger of its relative L2 error and its max-abs ratio, each over its bar."""
  return {k: max(r / bar(kind, prec, k)[0], m / bar(kind, prec, k)[1])
          for k, (r, m) in errors(kind, got, ref, V).items()}


# ---------------------------------------------------------------------------------------------------------------
# The inference forward (render_ray.net_dynamic_forward / net_static_forward): tests/test_staged_nets_gpu.py
# ---------------------------------------------------------------------------------------------------------------
# Planted errors of the inference forward (tests/test_staged_nets_reference_cpu.py).
FWD_PLANTS = (
    "pool2_first16",   # the second pooling (pool2_kernel) over the first 16 views only
    "keys_first256",   # the attention keys past the first 256 samples of a ray left out of its softmax
    "rays_chunk0",     # ray_dir / ref_rays of every internal chunk read from chunk 0 (the ray offset r0 dropped)
    "blend_first16",   # the static blending softmax (st_out_kernel) over the first 16 views only
)

HOT = 4.0  # weight scale of a "hot" case: pre-activations of several units, ELUs saturate at -1, sigmoids at 0 / 1


def make_forward_case(kind, R, S, V, aa=False, mrgb=False, hot=False, s_zero=False, seed=0, device="cpu"):
  """Seeded module (CPU, fp32) and inputs (fp32, on `device`) of one inference case, built like make_net_case.
  Points 0, 1 and 2 (flat over R S) see no view, only view 0 (a masked query row of the attention) and every view.
  mrgb: about 10 % of the source colours are exactly black, which mask_rgb masks out.  hot: every weight matrix
  but the LayerNorm's scaled by HOT.  s_zero: the anti-aliased pooling's s = 0, so that every view of a point has
  the same e_v and the pooling weights (e_v - min e) m_v are all 0."""
  from dynibar_b200 import mlp_network as nets, synthetic
  torch.manual_seed(seed)
  args = synthetic.make_args(int(aa), int(mrgb))
  if kind == "dynamic":
    mod = nets.DynibarDynamic(args, 32, S, shift=5.0)
  else:
    mod = nets.DynibarStatic(args, 32, S)
  with torch.no_grad():
    mod.out_geometry_fc[2].bias.fill_(1.0 if kind == "dynamic" else 0.5)
    if hot:
      for name, p in mod.named_parameters():
        if name.endswith(".weight") and "layer_norm" not in name:
          p.mul_(HOT)
    if s_zero:
      mod.s.zero_()
  g = torch.Generator(device=device).manual_seed(seed + 1)
  rn = lambda *shape: torch.randn(*shape, generator=g, device=device)
  ru = lambda *shape: torch.rand(*shape, generator=g, device=device)
  c = dict(kind=kind, aa=aa, mrgb=mrgb, mod=mod)
  c["pts"] = rn(R, S, 3) * 2
  feat = rn(R, S, V, 35)
  feat[..., :3] = ru(R, S, V, 3)
  if mrgb:
    feat[..., :3].masked_fill_(ru(R, S, V, 1) < 0.1, 0.0)
  mask = (ru(R, S, V, 1) > 0.3).float()
  mp = mask.view(R * S, V)
  mp[0] = 0.0
  mp[1] = 0.0
  mp[1, 0] = 1.0
  mp[2] = 1.0
  c["feat"], c["mask"] = feat, mask
  c["ray_dir"] = F.normalize(rn(R, 3), dim=-1)
  c["t"] = float(torch.tensor(0.4, dtype=torch.float32))
  c["ref_rays"] = rn(R, 6)
  c["src_rays"] = rn(R, S, V, 6)
  c["ray_diff"] = torch.cat([F.normalize(rn(R, S, V, 3), dim=-1), ru(R, S, V, 1) * 0.3 + 0.7], -1)
  return c


def forward(c, device, mode, lo=0, hi=None, plant=None, rays_per_chunk=None, dtype=torch.float64):
  """raw [hi - lo, S, 4] (float64) of rays [lo, hi) of case `c`, evaluated on `device` as one call.  plant
  "rays_chunk0" reads ray_dir / ref_rays of ray r at r mod rays_per_chunk.  dtype=torch.float32 evaluates the same
  arithmetic in float32 (see reference)."""
  hi = c["feat"].shape[0] if hi is None else hi
  d = lambda x: x[lo:hi].to(device, dtype, copy=True)
  rays = torch.arange(lo, hi)
  if plant == "rays_chunk0":
    rays = rays % rays_per_chunk
  per_ray = lambda x: x[rays.to(x.device)].to(device, dtype)
  w = {k: p.detach().to(device, dtype, copy=True) for k, p in c["mod"].named_parameters()}
  with torch.no_grad():
    if c["kind"] == "dynamic":
      return net_dynamic(w, d(c["pts"]), d(c["feat"]), per_ray(c["ray_dir"]), d(c["mask"]), c["t"],
                         float(c["mod"].shift), mode, plant)
    return net_static(w, d(c["pts"]), per_ray(c["ref_rays"]), d(c["src_rays"]), d(c["feat"]), d(c["ray_diff"]),
                      d(c["mask"]), c["aa"], c["mrgb"], mode, plant)


# Bars of raw in the inference comparison, per (net, precision): (relative L2 error, max |error| / max |reference|)
# over the entries that are not the -1e9 sentinel.  The cases with ordinary weights stay within the training
# comparison's bars of raw (BARS); the hot cases have their own.  How they were set is in
# tests/test_staged_nets_gpu.py; the comment beside each hot bar records the measured worst and its case.
FWD_BARS = {
    ("dynamic", "bf16"): BARS[("dynamic", "bf16")]["out"],
    ("dynamic", "fp32"): BARS[("dynamic", "fp32")]["out"],
    ("static", "bf16"): BARS[("static", "bf16")]["out"],
    ("static", "fp32"): BARS[("static", "fp32")]["out"],
}
FWD_HOT_BARS = {
    ("dynamic", "bf16"): (3e-03, 2e-02),  # 1.47e-03 5.03e-03 s193
    ("dynamic", "fp32"): (5e-05, 3e-04),  # 2.11e-05 1.46e-04 s193
    ("static", "bf16"): (2e-01, 6e-01),  # 5.60e-02 2.87e-01 s193
    ("static", "fp32"): (4e-05, 5e-05),  # 1.51e-05 2.39e-05 v24
}


def fwd_ratio(kind, prec, got, ref, hot=False):
  """The larger of raw's relative L2 error and max-abs ratio, each over its bar (inf when a sentinel differs)."""
  rel, mx = errors(kind, {"out": got}, {"out": ref})["out"]
  b = (FWD_HOT_BARS if hot else FWD_BARS)[(kind, prec)]
  return max(rel / b[0], mx / b[1]), (rel, mx)
