"""Host-side checks (no GPU) of the two memory formats the fused tensor-core kernels rely on:
the bf16 wgmma weight image (N-blocks, chunked, K-major 8x8 core matrices, folded bias, scale) built by
`fused_engine.cuh: append_layer`, and the activation tile image (`tile_image_off`)."""

import ctypes

import numpy as np
import pytest
import torch

from dynibar_b200 import _lib


def _bf16(x):
  return torch.from_numpy(np.asarray(x, dtype=np.float32)).to(torch.bfloat16).float().numpy()


def _pack(W, bias, Npad, colmap, scale, stage):
  N, Kw = W.shape
  Kpad = len(colmap)
  cm = np.ascontiguousarray(colmap, dtype=np.int32)
  out = np.zeros(Npad * Kpad * 2 + 64, dtype=np.uint8)
  nbytes, nch = ctypes.c_size_t(), ctypes.c_int()
  Wc = np.ascontiguousarray(W, dtype=np.float32)
  bc = None if bias is None else np.ascontiguousarray(bias, dtype=np.float32)
  rc = _lib.lib.dyn_debug_pack_layer(Wc.ctypes.data, None if bc is None else bc.ctypes.data, N, Kw, Npad, Kpad,
                                     cm.ctypes.data, scale, stage, out.ctypes.data, out.size,
                                     ctypes.byref(nbytes), ctypes.byref(nch))
  _lib.check(rc)
  return out[:nbytes.value].view(np.uint16), nch.value


def _blocks(Npad, Kpad, stage):
  """(first output, outputs, first k-step, k-steps) of every chunk, in image order"""
  out = []
  for n0 in range(0, Npad, 64):
    nb = min(64, Npad - n0)
    steps = min(stage // (nb * 32), 8)
    for k0 in range(0, Kpad // 16, steps):
      out.append((n0, nb, k0, min(steps, Kpad // 16 - k0)))
  return out


def _unpack(img16, Npad, Kpad, stage):
  """image -> dense [Npad, Kpad] fp32, following the layout documented in include/dynibar_b200.h"""
  dense = np.zeros((Npad, Kpad), dtype=np.float32)
  off = 0  # in bf16 elements
  for n0, nb, k0, ks in _blocks(Npad, Kpad, stage):
    for n in range(nb):
      for kk in range(ks * 16):
        byte = (kk // 8) * (nb * 16) + (n // 8) * 128 + (n % 8) * 16 + (kk % 8) * 2
        h = int(img16[off + byte // 2])
        dense[n0 + n, k0 * 16 + kk] = np.array([h << 16], dtype=np.uint32).view(np.float32)[0]
    off += nb * 16 * ks
  assert off == img16.size
  return dense


@pytest.mark.parametrize("N,Npad,Kw,Kpad,stage", [(256, 256, 103, 112, 16384), (35, 48, 256, 256, 16384),
                                                  (128, 128, 128, 128, 8192), (18, 32, 256, 256, 16384)])
def test_weight_image_layout_and_bias_fold(N, Npad, Kw, Kpad, stage):
  rng = np.random.default_rng(N + Kpad)
  W = rng.standard_normal((N, Kw)).astype(np.float32)
  b = rng.standard_normal(N).astype(np.float32)
  colmap = np.full(Kpad, -1, dtype=np.int32)
  perm = rng.permutation(Kw)[:min(Kw, Kpad - 2)]
  slots = rng.permutation(Kpad)
  colmap[slots[:len(perm)]] = perm
  hi_col, lo_col = int(slots[len(perm)]), int(slots[len(perm) + 1])
  colmap[hi_col], colmap[lo_col] = -2, -3
  scale = 1.4426950408889634
  img, nch = _pack(W, b, Npad, colmap, scale, stage)
  assert nch == len(_blocks(Npad, Kpad, stage))
  dense = _unpack(img, Npad, Kpad, stage)
  # weights: bf16(W * scale) in the mapped columns, zero elsewhere / in padded rows
  for k in range(Kpad):
    c = colmap[k]
    if c >= 0:
      np.testing.assert_array_equal(dense[:N, k], _bf16(W[:, c] * np.float32(scale)))
    elif c == -1:
      assert not dense[:, k].any()
  assert not dense[N:].any()
  # folded bias: hi + lo reproduces b * scale to 2^-16 relative
  bs = b * np.float32(scale)
  np.testing.assert_array_equal(dense[:N, hi_col], _bf16(bs))
  np.testing.assert_allclose(dense[:N, hi_col] + dense[:N, lo_col], bs, rtol=2.0 ** -15, atol=1e-30)
  # and the GEMM it encodes: operand with ones in the bias columns == W x + b (times scale), bf16 operands
  x = rng.standard_normal(Kw).astype(np.float32)
  a = np.zeros(Kpad, dtype=np.float32)
  for k in range(Kpad):
    if colmap[k] >= 0:
      a[k] = x[colmap[k]]
  a[hi_col] = a[lo_col] = 1.0
  got = dense[:N].astype(np.float64) @ _bf16(a).astype(np.float64)
  used = colmap[colmap >= 0]
  ref = (_bf16(W[:, used] * np.float32(scale)).astype(np.float64) @ _bf16(x[used]).astype(np.float64)) + bs
  np.testing.assert_allclose(got, ref, rtol=1e-4, atol=1e-4)


def test_pack_layer_rejects_bad_arguments():
  W = np.zeros((8, 16), dtype=np.float32)
  cm = np.zeros(16, dtype=np.int32)
  out = np.zeros(4096, dtype=np.uint8)
  nb, nc = ctypes.c_size_t(), ctypes.c_int()
  # Npad not a multiple of 16
  rc = _lib.lib.dyn_debug_pack_layer(W.ctypes.data, None, 8, 16, 24, 16, cm.ctypes.data, 1.0, 16384,
                                     out.ctypes.data, out.size, ctypes.byref(nb), ctypes.byref(nc))
  assert rc != 0 and b"dyn_debug_pack_layer" in _lib.lib.dyn_last_error()
  cm[3] = 99  # column out of range
  rc = _lib.lib.dyn_debug_pack_layer(W.ctypes.data, None, 8, 16, 16, 16, cm.ctypes.data, 1.0, 16384,
                                     out.ctypes.data, out.size, ctypes.byref(nb), ctypes.byref(nc))
  assert rc != 0


def test_tile_image_offsets():
  """rows x 8-column groups -> bytes: a bijection onto [0, tiles * KG * 2048) in 16-byte units, with
  the 32 rows of a warp contiguous (coalesced 512-byte stores) and whole tiles contiguous (one bulk copy)."""
  f = _lib.lib.dyn_debug_tile_image_off
  for KG in (16, 34):
    rows = 3 * 128
    offs = np.array([[f(r, g, KG) for g in range(KG)] for r in range(rows)], dtype=np.int64)
    assert (offs % 16 == 0).all()
    assert sorted(offs.ravel().tolist()) == list(range(0, rows * KG * 16, 16))
    for r0 in range(0, rows, 32):
      np.testing.assert_array_equal(offs[r0:r0 + 32, 5] - offs[r0, 5], 16 * np.arange(32))
    for t in range(3):
      blk = offs[128 * t:128 * (t + 1)]
      assert blk.min() == t * KG * 2048 and blk.max() == (t + 1) * KG * 2048 - 16
    # element (r, k): k-group stride 2048 inside a tile, as the wgmma descriptor (LBO = 2048, SBO = 128) expects
    assert f(5, 3, KG) - f(5, 2, KG) == 2048 and f(13, 0, KG) - f(5, 0, KG) == 128
