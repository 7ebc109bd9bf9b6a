"""Float64 reference of the bf16 MotionMLP kernel (csrc/motion_wg.cu).

MotionMLP.forward (mlp_network.py:605-618, the oracle's motion_mlp): PE(xyzt) with 16 linspace frequencies
(4 -> 132 columns), eight 256-wide ReLU layers with the skip cat([PE, h]) into pts_linears.5, and coeff_linear.
dyn_motion_coeffs also zeroes the last round(0.1 S) samples of each ray (the whole axis when that rounds to 0,
as Python's x[:, -0:] does), and render_ray divides by the module's sf_mag_div.

mode="exact" evaluates everything in float64 from the fp32 parameters.  mode="kernel" rounds where the kernel
rounds:
  - PE is evaluated in fp32 as the kernel does (sin / cos of x and of x * fp32(16/15), then the angle-addition
    recurrence) and handed on as bf16;
  - the weights are bf16(W); the biases stay fp32 and are added after the fp32 accumulation;
  - the hidden activations bf16(ReLU(a + b)) are the next layer's operand;
  - the coefficients are fp32 (acc + bias).

`plant` names a deliberate error (PLANTS) used to show that the tolerances of the GPU test would catch it.
"""

import torch

from oracle import dynibar_oracle as O

PLANTS = (
    "skip_no_pe",    # pts_linears.5 without its PE half
    "relu_skipped",  # no ReLU after pts_linears.4
    "bias_105",      # pts_linears.7 bias x 1.05
    "zero_short",    # one sample fewer zeroed at the end of each ray
)

# |got - ref| <= ATOL + MAG * mag + RTOL * |ref|, mag = sum_k |h_k W_nk| + |b_n| of coeff_linear (the scale of
# its fp32 accumulation and of the effect of a bf16 rounding flip of an upstream activation).  The largest
# flips come from PE at |x| in the tens, where the kernel's __sincosf and this fp32 sin / cos differ by more
# than elsewhere: the largest err / mag measured on an H100 is 1.75e-3, MAG is 2.2x that.
ATOL, MAG, RTOL = 0.0, 2.0 ** -8, 1e-6


def bf16(x):
  return x.to(torch.bfloat16).to(torch.float64)


def pe_kernel(xyzt):
  """PE(xyzt) [N,132] as the kernel computes it in fp32 (float64 tensor of bf16 values)."""
  x = xyzt.float()
  delta = torch.tensor(16.0 / 15.0, dtype=torch.float32)
  c, s = torch.cos(x), torch.sin(x)
  cd, sd = torch.cos(x * delta), torch.sin(x * delta)
  cs, ss = [], []
  for _ in range(16):
    cs.append(c)
    ss.append(s)
    c, s = c * cd - s * sd, s * cd + c * sd
  return bf16(torch.cat([x] + cs + ss, -1))


def motion_mlp(w, xyzt, mode="kernel", plant=None, div=1.0):
  """xyzt [N,4] -> {"coeff": [N,3 nb], "_mag": [N,3 nb]} (float64)."""
  k = mode == "kernel"
  p = lambda n: w[n].detach().to(xyzt.device, torch.float32)
  W = lambda n: bf16(p(n)) if k else p(n).double()
  r = lambda t: bf16(t) if k else t
  x0 = pe_kernel(xyzt) if k else O.periodic_embed(xyzt.double(), 16, linspace=True)
  h = x0
  for i in range(8):
    Wi, bi = W("pts_linears.%d.weight" % i), p("pts_linears.%d.bias" % i).double()
    if i == 7 and plant == "bias_105":
      bi = bi * 1.05
    if i == 5 and plant == "skip_no_pe":
      a = h[:, 132:] @ Wi[:, 132:].t() + bi
    else:
      a = h @ Wi.t() + bi
    h = a if (i == 4 and plant == "relu_skipped") else torch.relu(a)
    h = r(h)
    if i == 4:
      h = torch.cat([x0, h], -1)
  Wc, bc = W("coeff_linear.weight"), p("coeff_linear.bias").double()
  out = h @ Wc.t() + bc
  mag = h.abs() @ Wc.abs().t() + bc.abs()
  return {"coeff": out / div, "_mag": mag / abs(div)}


def n_last(S):
  """Samples zeroed at the end of each ray: int(round(0.1 S)), or all S when that is 0."""
  n = int(round(S * 0.1))
  return n if n > 0 else S


def motion_coeffs(w, pts, t, mode="kernel", plant=None, div=1.0):
  """pts [R,S,3], time t -> {"coeff": [R,S,3 nb], "_mag"} with the last samples of each ray zeroed."""
  R, S = pts.shape[:2]
  xyzt = torch.cat([pts.reshape(-1, 3).float(), torch.full((R * S, 1), float(t), device=pts.device)], -1)
  out = motion_mlp(w, xyzt, mode, plant, div)
  nl = n_last(S) - (1 if plant == "zero_short" else 0)
  keep = torch.ones(R, S, 1, dtype=torch.float64, device=pts.device)
  if nl > 0:
    keep[:, S - nl:] = 0.0
  return {"coeff": (out["coeff"].reshape(R, S, -1) * keep).reshape(R * S, -1), "_mag": out["_mag"]}


def errors(got, ref):
  """(max |got - ref|, max |got - ref| / tolerance, max (|got - ref| - RTOL |ref|) / mag).  Where the reference
  is zeroed the output must be exactly 0."""
  b = ref["coeff"]
  a = got.double().reshape(b.shape).to(b.device)
  mag = ref["_mag"].to(b.device)
  err = (a - b).abs()
  err = torch.where(torch.isnan(err), torch.full_like(err, float("inf")), err)
  zeroed = (b == 0) & (mag > 0)
  bound = ATOL + MAG * mag + RTOL * b.abs()
  ratio = torch.where(zeroed, torch.where(a == 0, 0.0, float("inf")), err / bound)
  per_mag = torch.where(zeroed, 0.0, (err - RTOL * b.abs()) / mag.clamp(min=1e-300))
  return float(err.max()), float(ratio.max()), float(per_mag.max())


def make_points(N, seed=0, scale=1.0, big=0):
  """Seeded sample points [N,3]: N(0, scale^2), the first `big` rows with |x| in the tens."""
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(N, 3, generator=g) * scale
  if big:
    x[:big] = (torch.rand(big, 3, generator=g) * 2 - 1) * 60.0
  return x
