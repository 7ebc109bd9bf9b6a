"""Float64 reference of the fused per-view stage (csrc/view_wg.cu) for a chosen subset of sample points.

The stage turns the points of one launch into what the per-point stage and the static blending head read:
G (pooled mean | variance | mean pooling weight, the bf16 operand of geometry_fc), nvalid, and for the static
net X (per-view features after the visibility residual, bf16), vis2, mask_eff, ray_diff and rgb_in.  Rows are
independent, so a large launch is checked on sampled points.

The formulas are the oracle's (oracle/dynibar_oracle.py: project_gather, plucker_*, periodic_embed,
_weighted_mean_var and the structure of _visibility_block), evaluated with float64 as the default dtype.  The
inputs are the ones the kernel reads: feature maps rounded to bf16, fp32 RGB, bf16 weights for every layer that
runs on the tensor cores and fp32 parameters elsewhere (biases, the visibility-logit row of vis_fc.2, vis_fc2.2,
ref_feature_fc, the dynamic net's time feature and the anti-alias sharpness s).

mode="exact" keeps float64 for every activation.  mode="kernel" rounds to bf16 exactly where view_wg.cu does:
  - the positional-encoding operand of ray_dir_fc.0 and each hidden activation that feeds the next layer;
  - the first-pooling operand [mean | var | feat] of base_fc.0;
  - x before vis_fc.0 (the pooling weight w1 scales the accumulator: w1 (W bf16(x)));
  - h before vis_fc.2 (the visibility logit is a float dot with the unrounded h);
  - x + res before vis_fc2.0 (vis1 scales the accumulator), which is also X as stored;
  - G as stored.
The pooling statistics, the logit dots and src_feat * ref_feat stay unrounded.  ref_feature_fc runs on the
fp32 SIMT linear (launch_linear in net_static_fused), so it uses the fp32 weights.

The twin-warp kernel (csrc/view_twin.cu) rounds at the same points but in other units: the hidden activations
of ray_dir_fc.0, base_fc.0, vis_fc.0 and vis_fc2.0 are handed on as bf16(log2(e) * ELU) with the consuming
weights scaled by ln(2) before their bf16 rounding, and the biases of base_fc.0, base_fc.2 and vis_fc.2 ride in
the MMA as a bf16 hi/lo pair (error 2^-17 |b|).  Its results therefore differ from mode="kernel" by about one
bf16 rounding per layer more than the warpgroup kernel's; the tolerances below cover both.

`plant` names a deliberate error (PLANTS) used to show that the tolerances of the GPU test would catch it.
"""

import contextlib

import torch
import torch.nn.functional as F

from oracle import dynibar_oracle as O

GCOLS = 272  # row stride of G: mean 0..127 | var 128..255 | W / V at 256 | bias columns 264, 265

# Planted errors (tests/test_view_stage_reference_cpu.py): each must move at least one compared output by
# at least 3x its tolerance.
PLANTS = (
    "var2_drop",        # second-pooling variance dropped
    "var2_scale",       # second-pooling variance x 1.05
    "vis0_over_V",      # vis_fc.0 input scaled by 1/V instead of the pooling weight
    "angle_neg",        # view-angle direction (ray_diff[:3]) negated
    "var1_drop",        # first-pooling variance dropped
    "chan_drop",        # one gathered feature channel dropped
    "view_swap",        # the gathered features of views 0 and 1 swapped
    "aa_min_masked",    # anti-alias minimum taken over masked-valid views only
    "no_time",          # dynamic net: time feature missing
    "ref_neighbor",     # static net: ref_feat of the neighbouring ray
    "mask_rgb_ignored", # mask_rgb test skipped
    "W_over_nvalid",    # the W / V column divided by the valid-view count instead of V
)

# Tolerances of the GPU comparison, per output (G per column block):
#   |got - ref| <= atol + ulps * ulp_bf16(ref) + cond * rd_cond
# ulps counts bf16 ulps of the reference value (bf16 outputs: the stored value may round the other way after
# fp32 summation-order differences).  atol covers bf16 rounding flips of hidden activations upstream; it is
# given per kernel (the warpgroup kernel, the twin-warp kernel, which rounds in other units) and for the "hot"
# case of the GPU test (per-view weights x3, where every layer's gain, and with it the effect of a flipped
# rounding, is larger).  Each atol is 1.5 - 3x the largest error beyond the ulps term measured on an H100
# across the GPU test's cases.  rd_cond = 1 / |a - b| is the conditioning of the normalised view-angle direction
# normalize(a - b), whose fp32 inputs carry an error of a few 2^-24.
ATOL_COLUMNS = ("wg", "twin", "wg_hot", "twin_hot")
TOL = {  # output: (atol per ATOL_COLUMNS, ulps, cond)
    "G_mean": ((3e-3, 5e-3, 4e-2, 1.5e-1), 1.0, 0.0),
    "G_var": ((3e-4, 1e-3, 1.5e-2, 8e-2), 1.0, 0.0),
    "G_w": ((0.0, 0.0, 0.0, 0.0), 1.0, 0.0),
    "X": ((4e-3, 5e-3, 4.5e-2, 2e-1), 1.0, 0.0),
    "vis2": ((1.5e-4, 3e-4, 1e-2, 2.5e-2), 0.0, 0.0),
    "nvalid": ((0.0, 0.0, 0.0, 0.0), 0.0, 0.0),
    "mask_eff": ((0.0, 0.0, 0.0, 0.0), 0.0, 0.0),
    "rgb_in": ((3e-5, 3e-5, 3e-5, 3e-5), 0.0, 0.0),
    "ray_diff": ((3e-6, 3e-6, 3e-6, 3e-6), 0.0, 2.0 ** -21),
}


@contextlib.contextmanager
def _float64():
  old = torch.get_default_dtype()
  torch.set_default_dtype(torch.float64)
  try:
    yield
  finally:
    torch.set_default_dtype(old)


def bf16(x):
  return x.to(torch.bfloat16).to(torch.float64)


def _lin(x, W, b=None):
  y = x @ W.t()
  return y if b is None else y + b


def blocks(G):
  """Column blocks of G compared with their own tolerances."""
  return {"G_mean": G[..., 0:128], "G_var": G[..., 128:256], "G_w": G[..., 256:GCOLS]}


def view_stage(kind, w, scene, idx=None, mode="kernel", plant=None):
  """The per-view stage of the static (kind="static") or dynamic net for points `idx` (all when None).

  w: the net's state_dict (fp32).  scene: dict with pts [P,3], S, query_cam [34], src_cams [V,34],
  src_rgbs [V,H,W,3], featmaps [V,32,h,w] (fp32; rounded to bf16 here), anti_alias, mask_rgb; static: ray_o,
  ray_d [R,3]; dynamic: pts_seq [V,P,3], time.  Returns float64 tensors: G [n,272], nvalid [n],
  mask_proj / mask_eff / vis2 [n,V], X [n,V,128], ray_diff [n,V,4], rgb_in [n,V,3], rd_cond [n,V,4] (1 / |a - b|
  of ray_diff's direction components, 0 for the dot product) and `ambiguous` [n,V]: views whose projector mask
  or mask_rgb test lies within rounding of its threshold."""
  assert mode in ("kernel", "exact") and (plant is None or plant in PLANTS)
  static = kind == "static"
  rnd = bf16 if mode == "kernel" else (lambda t: t)
  d = lambda t: t.detach().to("cpu", torch.float64)
  wb = lambda k: bf16(d(w[k]))  # tensor-core weights
  wf = lambda k: d(w[k])        # fp32 parameters
  with _float64():
    pts_all = d(scene["pts"])
    idx = torch.arange(pts_all.shape[0]) if idx is None else torch.as_tensor(idx, dtype=torch.long).cpu()
    pts = pts_all[idx]
    n = pts.shape[0]
    cams = d(scene["src_cams"])
    V = cams.shape[0]
    qcam = d(scene["query_cam"]).reshape(1, 34)
    xyz = d(scene["pts_seq"])[:, idx] if not static else pts[None].expand(V, n, 3)
    feats = bf16(d(scene["featmaps"]))
    rgbs = d(scene["src_rgbs"])

    # ---- projection, gather, masks, view-angle difference (projection.py:103-176) ----
    rgb_feat, rd, mask = O.project_gather(pts[:, None], xyz[:, :, None], qcam, rgbs[None], cams[None], feats)
    rgb_feat, rd, mask = rgb_feat[:, 0], rd[:, 0], mask[:, 0, :, 0]  # [n,V,35], [n,V,4], [n,V]
    pix, front = O.project_points(xyz, cams)
    Pm = cams[:, 2:18].reshape(-1, 4, 4).bmm(torch.inverse(cams[:, 18:34].reshape(-1, 4, 4)))
    z = xyz.bmm(Pm[:, 2, :3, None])[..., 0] + Pm[:, 2, 3:4]  # [V,n] depth in view v
    h_img, w_img = float(cams[0, 0]), float(cams[0, 1])
    edge = torch.stack([pix[..., 0].abs(), (pix[..., 0] - (w_img - 1)).abs(), pix[..., 1].abs(),
                        (pix[..., 1] - (h_img - 1)).abs()], -1).amin(-1)
    ambiguous = ((edge < 2e-3) | (z.abs() < 1e-6)).t().contiguous()  # [n,V]
    a = F.normalize(qcam[0, 18:34].reshape(4, 4)[:3, 3] - pts, dim=-1)[:, None]
    b = F.normalize(cams[:, 18:34].reshape(-1, 4, 4)[:, :3, 3][None] - xyz.transpose(0, 1), dim=-1)
    rd_cond = torch.cat([(1.0 / (a - b).norm(dim=-1, keepdim=True)).expand(-1, -1, 3), torch.zeros(n, V, 1)], -1)
    if plant == "angle_neg":
      rd = torch.cat([-rd[..., :3], rd[..., 3:]], -1)
    if plant == "chan_drop":
      rgb_feat = rgb_feat.clone()
      rgb_feat[..., 3 + 5] = 0
    if plant == "view_swap" and V > 1:
      rgb_feat = rgb_feat.clone()
      rgb_feat[:, [0, 1], 3:] = rgb_feat[:, [1, 0], 3:]
    rgb_in = rgb_feat[..., :3]
    mask_proj = mask
    if static and scene["mask_rgb"] and plant != "mask_rgb_ignored":
      srgb = rgb_in.sum(-1)
      mask = mask * (srgb > 1e-3).double()
      ambiguous |= (srgb - 1e-3).abs() < 1e-5

    if static:
      # ---- src_feat = ray_dir_fc([PE(pts), PE(plucker_src), ray_diff]); ref_feat per ray (:434-450) ----
      pl = O.plucker_src(pts[:, None], cams[None])[:, 0]  # [n,V,6]
      src_in = torch.cat([O.periodic_embed(pts, 5)[:, None].expand(-1, V, -1), O.periodic_embed(pl, 5), rd], -1)
      h1 = F.elu(_lin(rnd(src_in), wb("ray_dir_fc.0.weight"), wf("ray_dir_fc.0.bias")))
      src_feat = _lin(rnd(h1), wb("ray_dir_fc.2.weight"), wf("ray_dir_fc.2.bias"))
      R = scene["ray_o"].shape[0]
      ray = idx // scene["S"]
      if plant == "ref_neighbor":
        ray = (ray + 1) % R
      ref_pe = O.periodic_embed(O.plucker_ref(d(scene["ray_o"])[ray], d(scene["ray_d"])[ray]), 5)
      ref_feat = _lin(ref_pe, wf("ref_feature_fc.0.weight"), wf("ref_feature_fc.0.bias"))
      feat = torch.cat([rgb_feat, src_feat * ref_feat[:, None]], -1)  # 70
      if scene["anti_alias"]:
        e = torch.exp(wf("s").abs() * (rd[..., 3] - 1))
        pool = mask if plant == "aa_min_masked" else torch.ones_like(mask)
        emin = torch.where(pool > 0, e, torch.full_like(e, float("inf"))).amin(1, keepdim=True)
        emin = torch.where(torch.isinf(emin), torch.zeros_like(emin), emin)
        w1 = (e - emin) * mask
      else:
        w1 = mask.clone()
    else:
      # ---- + time feature (mlp_network.py:238-247), computed in fp32 by the library ----
      t_pe = O.periodic_embed(torch.tensor([[float(torch.tensor(scene["time"], dtype=torch.float32))]]), 10)
      dfeat = F.elu(_lin(F.elu(_lin(t_pe, wf("ray_dir_fc.0.weight"), wf("ray_dir_fc.0.bias"))),
                         wf("ray_dir_fc.2.weight"), wf("ray_dir_fc.2.bias")))
      feat = rgb_feat + (0 if plant == "no_time" else dfeat.reshape(1, 1, -1))
      w1 = mask.clone()
    w1 = w1 / (w1.sum(1, keepdim=True) + 1e-8)

    # ---- first pooling -> base_fc (mlp_network.py:248-270 / :461-483) ----
    mean, var = O._weighted_mean_var(feat[:, None], w1[:, None, :, None])
    mean, var = mean[:, 0], var[:, 0]  # [n,1,C]
    if plant == "var1_drop":
      var = torch.zeros_like(var)
    x = torch.cat([mean.expand(-1, V, -1), var.expand(-1, V, -1), feat], -1)
    h = F.elu(_lin(rnd(x), wb("base_fc.0.weight"), wf("base_fc.0.bias")))
    x = F.elu(_lin(rnd(h), wb("base_fc.2.weight"), wf("base_fc.2.bias")))

    # ---- visibility block (mlp_network.py:272-281 / :485-495; oracle _visibility_block) ----
    scale = torch.full_like(w1, 1.0 / V) if plant == "vis0_over_V" else w1
    h = F.elu(scale[..., None] * _lin(rnd(x), wb("vis_fc.0.weight")) + wf("vis_fc.0.bias"))
    W6, b6 = wf("vis_fc.2.weight"), wf("vis_fc.2.bias")
    logit = _lin(h, W6[128:129], b6[128:129])[..., 0]
    res = F.elu(_lin(rnd(h), bf16(W6[:128]), b6[:128]))
    vis1 = torch.sigmoid(F.elu(logit)) * mask
    x = x + res
    xs = rnd(x)
    h = F.elu(vis1[..., None] * _lin(xs, wb("vis_fc2.0.weight")) + wf("vis_fc2.0.bias"))
    vis2 = torch.sigmoid(_lin(h, wf("vis_fc2.2.weight"), wf("vis_fc2.2.bias"))[..., 0]) * mask

    # ---- second pooling -> G (the operand of geometry_fc) ----
    w2 = vis2 / (vis2.sum(1, keepdim=True) + 1e-8)
    mean2, var2 = O._weighted_mean_var(x[:, None], w2[:, None, :, None])
    mean2, var2 = mean2[:, 0, 0], var2[:, 0, 0]
    if plant == "var2_drop":
      var2 = torch.zeros_like(var2)
    if plant == "var2_scale":
      var2 = var2 * 1.05
    nvalid = mask.sum(1)
    wsum = w2.sum(1)
    wcol = wsum / nvalid.clamp(min=1) if plant == "W_over_nvalid" else wsum / V
    G = torch.zeros(n, GCOLS)
    G[:, 0:128], G[:, 128:256], G[:, 256] = mean2, var2, wcol
    G[:, 264:266] = 1.0
    return {"G": rnd(G), "nvalid": nvalid, "X": xs, "vis2": vis2, "mask_proj": mask_proj, "mask_eff": mask,
            "ray_diff": rd, "rgb_in": rgb_in, "ambiguous": ambiguous,
            "rd_cond": rd_cond}


# layers of the per-view stage (the tensor-core chain of view_wg.cu) whose weights make_case may scale
_PER_VIEW = {"static": ("ray_dir_fc.", "base_fc.", "vis_fc.", "vis_fc2."),
             "dynamic": ("base_fc.", "vis_fc.", "vis_fc2.")}


def make_case(V=8, rays=64, S=32, seed=0, H=72, W=96, stress=False, mask_rgb=0, anti_alias=1, s_zero=False,
              weight_scale=1.0, black=False, num_vv=0, far=30.0):
  """A seeded synthetic scene on the CPU -> (nets {"static", "dynamic"}, static scene, dynamic scene) in the
  form view_stage takes.  Both nets see V source views.  black: exact-black regions in the source images
  (the mask_rgb test fails there); s_zero: anti-alias sharpness |s| = 0 (every pooling weight is 0);
  weight_scale: multiplies the weights of the per-view layers (activations leave their near-linear range);
  num_vv: the last num_vv dynamic views are virtual views at the reference time (no displacement)."""
  from dynibar_b200 import synthetic
  batch, feat_c, _, _, t, _ = synthetic.make_scene(H=H, W=W, V_dy=V, V_st=V, rays=rays, seed=seed, stress=stress,
                                                   far=far)
  model, _ = synthetic.make_model(S, 0, args=synthetic.make_args(anti_alias, mask_rgb), seed=seed, mono=True)
  nets = {"static": model.net_coarse_st, "dynamic": model.net_coarse_dy}
  with torch.no_grad():
    if s_zero:
      nets["static"].s.zero_()
    for kind, net in nets.items():
      for name, p in net.named_parameters():
        if name.startswith(_PER_VIEW[kind]) and name.endswith(".weight"):
          p.mul_(weight_scale)
  g = torch.Generator().manual_seed(seed + 7)
  if black:
    for k in ("static_src_rgbs", "src_rgbs"):
      img = batch[k]
      img[:, :, : H // 2, : W // 3] = 0
      img[:, 1::2, H // 3:, W // 2:] = 0
  pts, _, _ = O.sample_along_ray(batch["ray_o"], batch["ray_d"], batch["depth_range"], S, True)
  seq = pts[None] + 0.02 * torch.randn(V, rays, S, 3, generator=g)
  if num_vv:
    seq[V - num_vv:] = pts[None]
  common = dict(pts=pts.reshape(-1, 3).contiguous(), S=S, query_cam=batch["camera"][0])
  st = dict(common, ray_o=batch["ray_o"], ray_d=batch["ray_d"], src_cams=batch["static_src_cameras"][0],
            src_rgbs=batch["static_src_rgbs"][0], featmaps=feat_c[2], anti_alias=bool(anti_alias),
            mask_rgb=bool(mask_rgb))
  dy = dict(common, pts_seq=seq.reshape(V, -1, 3).contiguous(), ray_d=batch["ray_d"],
            src_cams=batch["src_cameras"][0], src_rgbs=batch["src_rgbs"][0], featmaps=feat_c[0],
            time=float(t[0]), anti_alias=False, mask_rgb=False)
  return nets, st, dy


def ulp_bf16(x):
  """One bf16 ulp of x (0 at 0)."""
  m, e = torch.frexp(x.double())
  return torch.where(m != 0, torch.ldexp(torch.ones_like(m), e - 8), torch.zeros_like(m))


def errors(got, ref, kind, keep=None, column="wg"):
  """Per output the GPU test compares: (max |got - ref|, max |got - ref| / tolerance); the ratio is inf where
  the tolerance is 0 and the values differ.  got / ref: view_stage-shaped dicts; keep: points to compare;
  column: which atol of TOL (ATOL_COLUMNS)."""
  g, r = compared(got, kind), compared(ref, kind)
  out = {}
  for name in r:
    atols, ulps, kc = TOL[name]
    atol = atols[ATOL_COLUMNS.index(column)]
    a, b = g[name].double(), r[name].double()
    c = ref["rd_cond"] if name == "ray_diff" else torch.zeros_like(b)
    if keep is not None:
      a, b, c = a[keep], b[keep], c[keep]
    if b.numel() == 0:
      out[name] = (0.0, 0.0)
      continue
    err = (a - b).abs()
    bound = atol + ulps * ulp_bf16(b) + kc * c
    ratio = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, float("inf"), 0.0))
    out[name] = (float(err.max()), float(ratio.max()))
  return out


def compared(out, kind):
  """The outputs the GPU test compares for net `kind`, keyed by TOL name (the dynamic net writes G and
  nvalid only)."""
  c = dict(blocks(out["G"]))
  c["nvalid"] = out["nvalid"]
  if kind == "static":
    for k in ("X", "vis2", "mask_eff", "rgb_in", "ray_diff"):
      c[k] = out[k]
  return c
