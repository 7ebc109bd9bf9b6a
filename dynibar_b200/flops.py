"""Algorithmic work of the hot path, from the reference's layer widths
(SURVEY.md 8(a)/(d), App. A).  Padded-K work is NOT counted; work the
reference performs per (point, view) is counted per (point, view) even where a
kernel hoists it."""


def mac_per_point_view(kind):
  if kind == "dynamic":  # mlp_network.py:159-182
    return (21 * 256 + 256 * 35) + (105 * 256 + 256 * 128) + (128 * 128 + 128 * 129) + (128 * 128 + 128)
  if kind == "static":  # mlp_network.py:349-373, :388-394
    return ((103 * 256 + 256 * 35) + 66 * 35 + (210 * 256 + 256 * 128) + (128 * 128 + 128 * 129)
            + (128 * 128 + 128) + (261 * 128 + 128 * 64 + 64))
  raise ValueError(kind)


def mac_per_point(kind, S):
  attn = 4 * 128 * 128 + 2 * S * 128  # q,k,v,fc + QK^T + PV (mlp_network.py:56-104)
  geo = 257 * 256 + 256 * 128
  outgeo = 128 * 128 + 128
  if kind == "dynamic":  # + ref_pts_fc, rgb_fc (mlp_network.py:195-214)
    return geo + attn + (161 * 256 + 256 * 128) + outgeo + (155 * 128 + 128 * 64 + 64 * 3)
  if kind == "static":
    return geo + attn + outgeo
  if kind == "motion":  # mlp_network.py:591-601
    return 132 * 256 + 4 * 256 * 256 + 388 * 256 + 2 * 256 * 256 + 256 * 18
  raise ValueError(kind)


def rgbhead_bytes(points, V):
  """HBM bytes the static blending head (csrc/chains_wg.cu: rgbhead_wg_kernel) moves for `points` points with V
  source views: per view slot (VP = 8 for V <= 8, else 16) its 256-byte bf16 X row; per view vis2, mask_eff,
  ray_diff and rgb_in (36 B); per point its 512-byte fp32 GW row and sigma in, and raw (16 B) out.  The
  weights (54 KB per CTA) are not counted."""
  VP = 8 if V <= 8 else 16
  return points * (VP * 256 + V * 36 + 512 + 4 + 16)


def flop_per_ray(S_coarse, S_fine, V_dy, V_st):
  """2 * MAC over the coarse pass (S_coarse samples) and, when S_fine > 0, the
  fine pass (S_fine = N_samples + N_importance samples)."""
  total = 0
  for S in (S_coarse, S_fine):
    if S <= 0:
      continue
    per_pt = (mac_per_point("motion", S) + mac_per_point("dynamic", S) + mac_per_point("static", S)
              + V_dy * mac_per_point_view("dynamic") + V_st * mac_per_point_view("static"))
    total += 2 * S * per_pt
  return total
