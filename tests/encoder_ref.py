"""Float64 reference of the 2-D encoder's training forward and its backward (rows f1 / f2).

The library's training path (csrc/encoder.cu: dyn_encoder_train_forward, dyn_encoder_backward) runs the executed
part of ResNet.forward in fp32 SIMT kernels, keeps every convolution output, InstanceNorm statistic and activation,
and differentiates each convolution through its im2col form (ConvBwd::run):

  dYt [rows, 64]   = dY (NCHW) with rows = (n, oy, ox)
  col [rows, K]    = im2col(X) with the forward's reflect padding and stride, K = C_in k k, column = ci k k + ky k + kx
  dW  [64, K]      = dYt^T col                   (in 256-column chunks of K)
  dX               = col2im(dYt W)               (in 256-column chunks; a scatter-add through the same index map)
  d out_conv.bias  = column sum of dYt

and each InstanceNorm as enc_in_bwd_kernel does, with the plane statistics in float64:
  xh = (x - mean) rstd,  dx = rstd gamma (dy - mean(dy) - xh mean(dy xh)),  dgamma = sum dy xh,  dbeta = sum dy.

This module restates that computation.  The wiring is oracle.encoder_forward's; the convolutions and the
InstanceNorms go through the autograd Functions _Conv and _InstNorm below, whose backward is the library's written
out.  ReLU, the residual sums and the coarse / fine split are torch autograd.  Tensors may live on any device.

mode="exact" rounds nothing: the library's precision "fp32".  mode="kernel" rounds where precision "bf16" rounds
and nowhere else: a product that dispatch() puts on the tensor cores multiplies round-to-nearest bf16 copies of
both operands (dYt and col for dW, dYt and W for dX) and accumulates exactly.  The forward is fp32 SIMT in both
precisions, so it is exact in both modes.  dtype=torch.float32 evaluates the same arithmetic in float32 (CPU: no
TF32), which estimates how far the library's own fp32 arithmetic can drift from the float64 evaluation.

`plant` names a deliberate wiring error (PLANTS) used to show that the bars of the GPU test would catch it.
"""

import torch
import torch.nn.functional as F

# Planted wiring errors (tests/test_encoder_reference_cpu.py); each must move some compared tensor of the case it is
# scored on by at least MARGIN times its bf16 bar.
PLANTS = (
    "dw_ragged_tile",      # layer1.2.conv2's tensor-core dW leaves out the rows of the last, partial 128-row tile
    "in_drop_xh_term",     # layer1.1.bn1's InstanceNorm backward drops the - xh mean(dy xh) term
    "col2im_zero_pad",     # col2im drops what reaches the padding (the zero-padding adjoint, not the reflect one)
    "dx_drop_last_chunk",  # dX of every 3x3 convolution leaves out the last K chunk (columns 512..575)
    "b0_im2col_pad0",      # layer1.0.conv1 (stride 2) im2col / col2im with pad 0 instead of 1
    "bn_swap",             # layer1.1: bn1's dgamma / dbeta written to bn2's slots and bn2's to bn1's
    "d_fine_ignored",      # the fine half of the upstream gradient is dropped
    "ds_dx_overwrite",     # the shortcut conv's dX overwrites d a1 instead of adding to conv1's (zero_dx = true)
)

# a ReLU pre-activation z = IN(conv(x)) [+ shortcut] counts as "near 0" when |z| <= RELU_NEAR times the magnitude its
# rounding error scales with (_Enc.scale: the convolution's terms and the plane mean in absolute value, through the
# normalisation): about 256 fp32 ulps of that scale, where the fp32 / float64 difference of the forward can put it on
# the other side of the kink
RELU_NEAR = 2.0 ** -16


def bf16(x):
  return x.to(torch.bfloat16).to(x.dtype)


def dims(H, W):
  """(H2, W2, H4, W4): half resolution after the stem, quarter resolution after layer1.0 (enc_dims)."""
  H2, W2 = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
  return H2, W2, (H2 + 2 - 3) // 2 + 1, (W2 + 2 - 3) // 2 + 1


# ---------------------------------------------------------------------------------------------------------------
# Dispatch: which product runs on the tensor cores.  ConvBwd::run (csrc/encoder.cu:387-397 dW, :399-409 dX) splits
# K into 256-column chunks and asks tc_grad_w_ok / tc_grad_in_ok (csrc/train_tc.cu:179-180) per chunk, with
# out = 64: bf16 and rows >= 2048 (tc_grad_in_ok also wants width >= 16; every chunk here has 64, 147 or 256
# columns).  Everything else (IN, ReLU, im2col / col2im, the bias column sum) is fp32 SIMT in both precisions.
# ---------------------------------------------------------------------------------------------------------------
def dispatch(prec, rows, width):
  """Column chunks [(c0, c1, on_tensor_cores)] of one convolution's dW or dX product over `rows` rows of dYt and
  `width` = K columns, in precision `prec`."""
  out = []
  for c0 in range(0, width, 256):
    c1 = min(width, c0 + 256)
    out.append((c0, c1, prec == "bf16" and rows >= 2048 and c1 - c0 >= 16))
  return out


def _reflect(i, n):
  """enc_im2col_kernel's reflect_idx on an index tensor, and whether the position lies inside the image."""
  inside = (i >= 0) & (i < n)
  j = torch.where(i < 0, -i, i)
  j = torch.where(j >= n, 2 * n - 2 - j, j)
  return j.clamp(0, n - 1), inside


def _maps(n_in, n_out, k, stride, pad, device):
  """Per output position o and tap t: the input index reflect(o stride + t - pad) [n_out, k], and inside-ness."""
  i = torch.arange(n_out, device=device)[:, None] * stride + torch.arange(k, device=device)[None, :] - pad
  return _reflect(i, n_in)


def im2col(X, k, stride, pad, Ho, Wo):
  """col [N Ho Wo, C k k]: row (n, oy, ox), column ci k k + ky k + kx."""
  N, C, H, W = X.shape
  iy, _ = _maps(H, Ho, k, stride, pad, X.device)
  ix, _ = _maps(W, Wo, k, stride, pad, X.device)
  g = X[:, :, iy][:, :, :, :, ix]                       # [N, C, Ho, ky, Wo, kx]
  return g.permute(0, 2, 4, 1, 3, 5).reshape(N * Ho * Wo, C * k * k)


def col2im(dcol, shape, k, stride, pad, Ho, Wo, zero_pad=False):
  """The adjoint of im2col: scatter-add of dcol through the same index map.  zero_pad: positions outside the image
  are dropped instead of reflected (the adjoint of zero padding; a planted error)."""
  N, C, H, W = shape
  iy, in_y = _maps(H, Ho, k, stride, pad, dcol.device)
  ix, in_x = _maps(W, Wo, k, stride, pad, dcol.device)
  g = dcol.reshape(N, Ho, Wo, C, k, k).permute(0, 3, 1, 4, 2, 5)  # [N, C, Ho, ky, Wo, kx]
  if zero_pad:
    g = g * (in_y[:, :, None, None] & in_x[None, None]).to(g.dtype)
  t = g.new_zeros(N, C, H, Wo, k).index_add_(2, iy.reshape(-1), g.reshape(N, C, Ho * k, Wo, k))
  return g.new_zeros(N, C, H, W).index_add_(3, ix.reshape(-1), t.reshape(N, C, H, Wo * k))


class _Spec(object):
  """One layer: its name, rounding on / off, precision of the dispatch, plant, ReLU statistics."""

  def __init__(self, name, kernel, plant, stats, k=1, stride=1, pad=0):
    self.name, self.k, self.plant, self.stats = name, kernel, plant, stats
    self.ks, self.stride, self.pad = k, stride, pad


class _Conv(torch.autograd.Function):
  """Y = conv2d(reflect_pad(X), W) (+ b); backward as ConvBwd::run."""

  @staticmethod
  def forward(ctx, sp, X, W, b):
    Xp = F.pad(X, (sp.pad,) * 4, mode="reflect") if sp.pad else X
    Y = F.conv2d(Xp, W, b, stride=sp.stride)
    ctx.sp = sp
    ctx.save_for_backward(X, W)
    return Y

  @staticmethod
  def backward(ctx, dY):
    sp = ctx.sp
    X, W = ctx.saved_tensors
    N, Co, Ho, Wo = dY.shape
    rows, K = N * Ho * Wo, W[0].numel()
    pad = 0 if (sp.plant == "b0_im2col_pad0" and sp.name == "layer1.0.conv1") else sp.pad
    prec = "bf16" if sp.k else "fp32"
    dYt = dY.permute(0, 2, 3, 1).reshape(rows, Co)
    col = im2col(X, sp.ks, sp.stride, pad, Ho, Wo)
    W2 = W.reshape(Co, K)
    dW = W2.new_zeros(Co, K)
    for c0, c1, tc in dispatch(prec, rows, K):
      A, B = dYt, col[:, c0:c1]
      if tc:
        A, B = bf16(A), bf16(B)
        if sp.plant == "dw_ragged_tile" and sp.name == "layer1.2.conv2" and rows % 128:
          A, B = A[:rows - rows % 128], B[:rows - rows % 128]
      dW[:, c0:c1] = A.t() @ B
    db = dYt.sum(0) if ctx.needs_input_grad[3] else None
    dX = None
    if ctx.needs_input_grad[1]:
      dcol = col.new_zeros(rows, K)
      for c0, c1, tc in dispatch(prec, rows, K):
        if sp.plant == "dx_drop_last_chunk" and sp.ks == 3 and c0 == 512:
          continue
        A, B = (bf16(dYt), bf16(W2[:, c0:c1])) if tc else (dYt, W2[:, c0:c1])
        dcol[:, c0:c1] = A @ B
      dX = col2im(dcol, X.shape, sp.ks, sp.stride, pad, Ho, Wo, zero_pad=sp.plant == "col2im_zero_pad")
      if sp.plant == "ds_dx_overwrite" and sp.name == "layer1.0.conv1":
        dX = torch.zeros_like(dX)  # the shortcut's col2im lands on a zeroed d a1 after conv1's
    return None, dX, dW.reshape(W.shape), db


class _InstNorm(torch.autograd.Function):
  """InstanceNorm2d(affine), eps 1e-5, biased variance; backward as enc_in_bwd_kernel."""

  @staticmethod
  def forward(ctx, sp, x, gamma, beta):
    m = x.mean((2, 3), keepdim=True)
    var = ((x - m) ** 2).mean((2, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    xh = (x - m) * rstd
    ctx.sp = sp
    ctx.save_for_backward(xh, rstd, gamma)
    return xh * gamma[:, None, None] + beta[:, None, None]

  @staticmethod
  def backward(ctx, dy):
    sp = ctx.sp
    xh, rstd, gamma = ctx.saved_tensors
    mg = dy.mean((2, 3), keepdim=True)
    mgx = (dy * xh).mean((2, 3), keepdim=True)
    if sp.plant == "in_drop_xh_term" and sp.name == "layer1.1.bn1":
      mgx = torch.zeros_like(mgx)
    dx = rstd * gamma[:, None, None] * (dy - mg - xh * mgx)
    return None, dx, (dy * xh).sum((0, 2, 3)), dy.sum((0, 2, 3))


class _Enc(object):
  def __init__(self, w, mode, plant, stats):
    assert mode in ("exact", "kernel")
    self.w, self.k, self.plant, self.stats = w, mode == "kernel", plant, stats

  def conv(self, name, x, k, stride, pad, bias=False):
    sp = _Spec(name, self.k, self.plant, self.stats, k, stride, pad)
    return _Conv.apply(sp, x, self.w[name + ".weight"], self.w[name + ".bias"] if bias else None)

  def norm(self, name, x):
    g, b = self.w[name + ".weight"], self.w[name + ".bias"]
    if self.plant == "bn_swap" and name in ("layer1.1.bn1", "layer1.1.bn2"):
      o = "layer1.1.bn2" if name == "layer1.1.bn1" else "layer1.1.bn1"
      g, b = _Swap.apply(g, self.w[o + ".weight"]), _Swap.apply(b, self.w[o + ".bias"])
    return _InstNorm.apply(_Spec(name, self.k, self.plant, self.stats), x, g, b)

  def scale(self, name, x, k, stride, pad, y):
    """The magnitude an InstanceNorm output's rounding error scales with: |gamma| rstd (sum |w x| + |mean|) + |beta|
    for y = IN(conv(x)), the convolution's terms in absolute value (None when no statistics are kept)."""
    if self.stats is None:
      return None
    with torch.no_grad():
      xp = F.pad(x, (pad,) * 4, mode="reflect") if pad else x
      mag = F.conv2d(xp.abs(), self.w[name + ".weight"].abs(), stride=stride)
      m = y.mean((2, 3), keepdim=True)
      rstd = 1.0 / torch.sqrt(((y - m) ** 2).mean((2, 3), keepdim=True) + 1e-5)
      bn = name.replace("conv", "bn").replace("downsample.0", "downsample.1")
      return (self.w[bn + ".weight"].abs()[:, None, None] * rstd * (mag + m.abs())
              + self.w[bn + ".bias"].abs()[:, None, None])

  def relu(self, name, z, scale):
    if self.stats is not None:
      with torch.no_grad():
        self.stats[name] = (int((z.abs() <= RELU_NEAR * scale).sum()), z.numel())
    return torch.relu(z)


class _Swap(torch.autograd.Function):
  """Forward: a; backward: the gradient of a goes to b (a planted wiring error of the parameter slots)."""

  @staticmethod
  def forward(ctx, a, b):
    return a.clone()

  @staticmethod
  def backward(ctx, g):
    return None, g


def encoder(w, x, mode="kernel", plant=None, stats=None):
  """oracle.encoder_forward through the library's backward: w {name: tensor} (the _EXECUTED parameters),
  x [N,3,H,W] -> (coarse, fine).  `stats`, a dict, receives per ReLU (pre-activations near 0, all of them)."""
  n = _Enc(w, mode, plant, stats)
  y = n.conv("conv1", x, 7, 2, 3)
  x = n.relu("bn1", n.norm("bn1", y), n.scale("conv1", x, 7, 2, 3, y))
  for b in range(3):
    p = "layer1.%d." % b
    s = 2 if b == 0 else 1
    y = n.conv(p + "conv1", x, 3, s, 1)
    out = n.relu(p + "bn1", n.norm(p + "bn1", y), n.scale(p + "conv1", x, 3, s, 1, y))
    y = n.conv(p + "conv2", out, 3, 1, 1)
    sc = n.scale(p + "conv2", out, 3, 1, 1, y)
    out = n.norm(p + "bn2", y)
    ident = x
    if b == 0:
      y = n.conv(p + "downsample.0", x, 1, 2, 0)
      sc = None if sc is None else sc + n.scale(p + "downsample.0", x, 1, 2, 0, y)
      ident = n.norm(p + "downsample.1", y)
    elif sc is not None:
      sc = sc + ident.abs()
    x = n.relu(p + "bn2", out + ident, sc)
  out = n.conv("out_conv", x, 1, 1, 0, bias=True)
  return out[:, :32], out[:, 32:]


# ---------------------------------------------------------------------------------------------------------------
# Cases and comparison, shared by the CPU and GPU tests
# ---------------------------------------------------------------------------------------------------------------
# name: (N, H, W, gradient) with gradient "both", "coarse" or "fine"; rows of the half / quarter resolution
# products in the comments (N H2 W2 / N H4 W4)
CASES = {
    "minimum": (1, 8, 8, "both"),          # 16 / 4: 2-wide planes under reflect padding, all SIMT
    "small_odd": (3, 17, 33, "both"),      # 459 / 135: odd sizes under stride 2, tile loads past the image
    "mixed": (2, 72, 96, "both"),          # 3456 / 864: stem on the tensor cores, quarter resolution in SIMT
    "below_2048": (1, 90, 354, "both"),    # 7965 / 2047: one row under the threshold
    "at_2048": (2, 128, 128, "fine"),      # 8192 / 2048: at the threshold, no partial tile
    "ragged": (3, 150, 206, "both"),       # 23175 / 5928: partial last 128-row tile at both resolutions
    "flat": (2, 64, 96, "both"),           # 3072 / 768: constant images, InstanceNorm variance near 0
    "bench": (8, 288, 512, "coarse"),      # 294912 / 73728: bench.py's train_step call
}


def make_model(seed):
  """fn.ResNet with non-trivial InstanceNorm affines and biases (the defaults are 1 / 0)."""
  from dynibar_b200 import feature_network as fn
  torch.manual_seed(seed)
  m = fn.ResNet()
  with torch.no_grad():
    for name, p in m.named_parameters():
      if name.endswith("bn1.weight") or name.endswith("bn2.weight") or name.endswith("downsample.1.weight"):
        p.uniform_(0.5, 1.5)
      elif name.endswith(".bias"):
        p.uniform_(-0.3, 0.3)
  return m.requires_grad_(False)


def make_case(name, seed=0):
  """Seeded module, images [N,3,H,W] (CPU, fp32) and upstream gradients (None where the loss ignores an output) of
  one case of CASES."""
  N, H, W, which = CASES[name]
  s = seed + N * 1000 + H
  g = torch.Generator().manual_seed(s + 1)
  x = torch.rand(N, 3, H, W, generator=g)
  if name == "flat":
    x[0] = 0.4
    x[1] = 0.6 + 1e-4 * torch.randn(3, H, W, generator=g)
  h, w = dims(H, W)[2:]
  gc = torch.randn(N, 32, h, w, generator=g) if which in ("both", "coarse") else None
  gf = torch.randn(N, 32, h, w, generator=g) if which in ("both", "fine") else None
  return dict(name=name, mod=make_model(s), x=x, gc=gc, gf=gf)


def executed_params(mod):
  from dynibar_b200 import feature_network as fn
  sd = mod.state_dict()
  return {k: sd[k] for k in fn._EXECUTED}


def reference(c, device, mode="kernel", plant=None, stats=None, dtype=torch.float64):
  """Coarse, fine and every executed parameter's gradient of case `c` on `device`:
  {"coarse", "fine", "<param>": d param}."""
  d = lambda t: t.detach().to(device, dtype, copy=True)
  w = {k: d(p).requires_grad_(True) for k, p in executed_params(c["mod"]).items()}
  co, fi = encoder(w, d(c["x"]), mode, plant, stats)
  loss = 0.0
  if c["gc"] is not None:
    loss = loss + (co * d(c["gc"])).sum()
  if c["gf"] is not None and plant != "d_fine_ignored":
    loss = loss + (fi * d(c["gf"])).sum()
  loss.backward()
  res = {"coarse": co.detach(), "fine": fi.detach()}
  res.update({k: v.grad for k, v in w.items()})
  return res


# Bars of the GPU comparison: per precision and compared tensor, (relative L2 error, max |error| / max |reference|),
# over every case but "flat" (FLAT_BAR).  How they were set is in tests/test_encoder_train_gpu.py; beside each bar the
# measured worst relative L2 error and max-abs ratio and the case that gave them.
BARS = {
    "bf16": {
        "bn1.bias": (1e-02, 2e-02),  # 4.77e-03 5.48e-03 below_2048
        "bn1.weight": (2e-02, 1e-02),  # 5.33e-03 4.86e-03 below_2048
        "coarse": (1e-04, 1e-04),  # 5.80e-06 7.93e-06 minimum
        "conv1.weight": (1e-02, 1e-02),  # 4.56e-03 4.75e-03 below_2048 / bench
        "fine": (1e-04, 1e-04),  # 4.91e-06 4.99e-06 minimum
        "layer1.0.bn1.bias": (8e-03, 2e-02),  # 3.89e-03 5.36e-03 below_2048
        "layer1.0.bn1.weight": (9e-03, 2e-02),  # 4.16e-03 5.29e-03 below_2048
        "layer1.0.bn2.bias": (9e-03, 2e-02),  # 4.12e-03 5.74e-03 below_2048
        "layer1.0.bn2.weight": (9e-03, 2e-02),  # 4.32e-03 5.62e-03 below_2048
        "layer1.0.conv1.weight": (9e-03, 1e-02),  # 4.19e-03 4.67e-03 below_2048
        "layer1.0.conv2.weight": (9e-03, 2e-02),  # 4.08e-03 5.40e-03 below_2048
        "layer1.0.downsample.0.weight": (9e-03, 2e-02),  # 4.16e-03 6.03e-03 below_2048
        "layer1.0.downsample.1.bias": (9e-03, 2e-02),  # 4.12e-03 5.74e-03 below_2048
        "layer1.0.downsample.1.weight": (8e-03, 2e-02),  # 3.82e-03 6.52e-03 below_2048
        "layer1.1.bn1.bias": (7e-03, 7e-03),  # 3.42e-03 3.43e-03 below_2048
        "layer1.1.bn1.weight": (8e-03, 1e-02),  # 3.59e-03 4.89e-03 below_2048
        "layer1.1.bn2.bias": (6e-03, 5e-03),  # 2.59e-03 2.14e-03 below_2048
        "layer1.1.bn2.weight": (7e-03, 9e-03),  # 3.34e-03 4.17e-03 below_2048
        "layer1.1.conv1.weight": (8e-03, 1e-02),  # 3.98e-03 4.81e-03 below_2048
        "layer1.1.conv2.weight": (8e-03, 1e-02),  # 3.92e-03 4.91e-03 below_2048
        "layer1.2.bn1.bias": (2e-02, 5e-02),  # 6.65e-03 2.10e-02 below_2048
        "layer1.2.bn1.weight": (2e-03, 2e-03),  # 5.44e-04 9.30e-04 bench / below_2048
        "layer1.2.bn2.bias": (9e-04, 3e-03),  # 4.35e-04 1.39e-03 bench
        "layer1.2.bn2.weight": (1e-03, 4e-03),  # 4.71e-04 1.51e-03 bench
        "layer1.2.conv1.weight": (1e-02, 5e-02),  # 4.98e-03 2.42e-02 below_2048
        "layer1.2.conv2.weight": (2e-03, 6e-03),  # 5.02e-04 2.66e-03 bench
        "out_conv.bias": (1e-04, 1e-04),  # 3.36e-07 3.63e-07 bench / below_2048
        "out_conv.weight": (2e-04, 6e-04),  # 7.90e-05 2.72e-04 at_2048
    },
    "fp32": {
        "bn1.bias": (1e-02, 2e-02),  # 4.77e-03 5.48e-03 below_2048
        "bn1.weight": (2e-02, 1e-02),  # 5.33e-03 4.86e-03 below_2048
        "coarse": (2e-05, 2e-05),  # 5.80e-06 7.93e-06 minimum
        "conv1.weight": (9e-03, 1e-02),  # 4.22e-03 4.85e-03 below_2048
        "fine": (1e-05, 1e-05),  # 4.91e-06 4.99e-06 minimum
        "layer1.0.bn1.bias": (8e-03, 2e-02),  # 3.89e-03 5.36e-03 below_2048
        "layer1.0.bn1.weight": (9e-03, 2e-02),  # 4.16e-03 5.29e-03 below_2048
        "layer1.0.bn2.bias": (9e-03, 2e-02),  # 4.12e-03 5.74e-03 below_2048
        "layer1.0.bn2.weight": (9e-03, 2e-02),  # 4.32e-03 5.62e-03 below_2048
        "layer1.0.conv1.weight": (9e-03, 1e-02),  # 4.19e-03 4.67e-03 below_2048
        "layer1.0.conv2.weight": (9e-03, 2e-02),  # 4.08e-03 5.40e-03 below_2048
        "layer1.0.downsample.0.weight": (9e-03, 2e-02),  # 4.16e-03 6.03e-03 below_2048
        "layer1.0.downsample.1.bias": (9e-03, 2e-02),  # 4.12e-03 5.74e-03 below_2048
        "layer1.0.downsample.1.weight": (8e-03, 2e-02),  # 3.82e-03 6.52e-03 below_2048
        "layer1.1.bn1.bias": (7e-03, 7e-03),  # 3.42e-03 3.43e-03 below_2048
        "layer1.1.bn1.weight": (8e-03, 1e-02),  # 3.59e-03 4.89e-03 below_2048
        "layer1.1.bn2.bias": (6e-03, 5e-03),  # 2.59e-03 2.14e-03 below_2048
        "layer1.1.bn2.weight": (7e-03, 9e-03),  # 3.34e-03 4.17e-03 below_2048
        "layer1.1.conv1.weight": (8e-03, 1e-02),  # 3.98e-03 4.81e-03 below_2048
        "layer1.1.conv2.weight": (8e-03, 1e-02),  # 3.92e-03 4.91e-03 below_2048
        "layer1.2.bn1.bias": (2e-02, 5e-02),  # 6.65e-03 2.10e-02 below_2048
        "layer1.2.bn1.weight": (2e-03, 2e-03),  # 5.36e-04 9.30e-04 bench / below_2048
        "layer1.2.bn2.bias": (9e-04, 3e-03),  # 4.33e-04 1.39e-03 bench
        "layer1.2.bn2.weight": (1e-03, 4e-03),  # 4.70e-04 1.50e-03 bench
        "layer1.2.conv1.weight": (1e-02, 5e-02),  # 4.98e-03 2.42e-02 below_2048
        "layer1.2.conv2.weight": (1e-03, 6e-03),  # 4.91e-04 2.63e-03 bench
        "out_conv.bias": (1e-05, 1e-05),  # 3.57e-07 3.63e-07 bench / below_2048
        "out_conv.weight": (1e-05, 3e-05),  # 4.76e-06 1.08e-05 minimum
    },
}

# Case "flat": only coarse and fine are compared (and every gradient must be finite); tests/test_encoder_train_gpu.py
# says why.  2x the worst measured: coarse 2.72e-03 2.69e-03, fine 2.57e-03 2.76e-03, both precisions.
FLAT_BAR = (6e-03, 6e-03)


def bar(prec, name):
  return BARS[prec][name]


def errors(got, ref):
  """{name: (relative L2 error, max |error| / max |ref|)} over every tensor of `ref`."""
  out = {}
  for name, b in ref.items():
    b = b.double()
    a = got[name].detach().to(b.device, torch.float64).reshape(b.shape)
    e = a - b
    nb, mb = float(b.norm()), float(b.abs().max())
    out[name] = (float(e.norm()) / nb if nb > 0 else float(e.norm()),
                 float(e.abs().max()) / mb if mb > 0 else float(e.abs().max()))
  return out


def ratios(prec, got, ref, flat=False):
  """Per tensor: the larger of its relative L2 error and its max-abs ratio, each over its bar (FLAT_BAR for case
  "flat")."""
  b = (lambda k: FLAT_BAR) if flat else (lambda k: bar(prec, k))
  return {k: max(r / b(k)[0], m / b(k)[1]) for k, (r, m) in errors(got, ref).items()}
