"""A harness that checks the library's memory contract (include/dynibar_b200.h, "Conventions"): an entry point writes
only inside the workspace and output extents it declares, and reads nothing it did not write first.

Under `poisoned(pattern)`:
  - `_lib.workspace` is a strict workspace: every `get(nbytes, device, slot)` returns a fresh allocation of exactly
    `nbytes` bytes (the leading view of a buffer of nbytes rounded up to 256 plus a 64 KiB guard band; the base keeps
    torch's 512-byte alignment), the whole buffer filled with the pattern byte.
  - `torch.empty` and `torch.empty_like` of a CUDA tensor return the leading elements of a buffer with a 64 KiB guard
    tail, all of it filled with the pattern byte.  This covers the wrappers' outputs, the autograd `saved` buffers,
    the PackedNet images and the scene loaders' device buffers.  Host and pinned tensors are left alone, and so is
    memory obtained any other way (torch.zeros, torch.full, the library's own cudaMalloc).
  - on exit, after a device synchronise, every byte from each buffer's declared end to its real end (rounding slack
    included) must still hold the pattern.

The guards are bytes past the declared size, never in place of it, and no base pointer moves: the harness cannot make a
correct kernel fault.  Three patterns: 0x00; 0xFF, NaN in fp32 and bf16; 0x7F, 3.39e38 in fp32 and bf16, finite, so a
product with a stale element that should have been multiplied by 0 turns into inf in any sum.  Outputs that must not
depend on the previous contents of memory are then compared across the patterns."""

import contextlib

import pytest
import torch

from dynibar_b200 import _lib

PATTERNS = (0x00, 0xFF, 0x7F)
GUARD = 64 << 10
ALIGN = 256


class Poison(object):
  def __init__(self, pattern):
    self.pattern = pattern
    self.bufs = []  # (uint8 buffer, declared bytes, what)
    self.real_empty = torch.empty
    self.real_empty_like = torch.empty_like

  def _buffer(self, nbytes, device, what):
    buf = self.real_empty(-(-nbytes // ALIGN) * ALIGN + GUARD, dtype=torch.uint8, device=device)
    buf.fill_(self.pattern)
    self.bufs.append((buf, nbytes, what))
    return buf

  # ---- the strict workspace ----
  def get(self, nbytes, device, slot=0):
    nbytes = int(nbytes)
    return self._buffer(nbytes, device, "workspace slot %r (%d bytes)" % (slot, nbytes))[:nbytes]

  # ---- poisoned device allocations ----
  def _tensor(self, shape, dtype, device):
    shape = torch.Size(shape)
    nbytes = shape.numel() * dtype.itemsize
    buf = self._buffer(nbytes, device, "torch.empty(%s, %s) (%d bytes)" % (tuple(shape), dtype, nbytes))
    t = self.real_empty(0, dtype=dtype, device=device)
    return t.set_(buf.untyped_storage(), 0, shape)

  @staticmethod
  def _plain(kw):
    return (kw.get("out") is None and not kw.get("pin_memory") and not kw.get("requires_grad")
            and kw.get("memory_format") in (None, torch.contiguous_format, torch.preserve_format))

  def empty(self, *size, **kw):
    dev = kw.get("device")
    if dev is None or torch.device(dev).type != "cuda" or not self._plain(kw):
      return self.real_empty(*size, **kw)
    shape = size[0] if len(size) == 1 and not isinstance(size[0], int) else size
    return self._tensor(shape, kw.get("dtype") or torch.get_default_dtype(), torch.device(dev))

  def empty_like(self, x, **kw):
    dev = torch.device(kw.get("device") or x.device)
    if dev.type != "cuda" or not self._plain(kw) or not x.is_contiguous():
      return self.real_empty_like(x, **kw)
    return self._tensor(x.shape, kw.get("dtype") or x.dtype, dev)

  def check(self):
    torch.cuda.synchronize()
    bad = []
    for buf, n, what in self.bufs:
      tail = buf[n:]
      hit = (tail != self.pattern).nonzero()
      if hit.numel():
        bad.append("%s: %d guard bytes changed, the first at declared end + %d" % (what, hit.numel(), hit[0].item()))
    assert not bad, "pattern 0x%02X: writes past the declared end of %d buffer(s):\n  %s" % (
        self.pattern, len(bad), "\n  ".join(bad))


def drop_packed(*objs):
  """Forget the cached PackedNet of every network module in `objs` (modules, or namespaces holding modules), so the
  next call packs its weights again into a poisoned buffer."""
  for o in objs:
    mods = [o] if isinstance(o, torch.nn.Module) else [v for v in vars(o).values() if isinstance(v, torch.nn.Module)]
    for m in mods:
      for sub in m.modules():
        for k in [k for k in sub.__dict__ if k.startswith("_dyn_pack_cache")]:
          del sub.__dict__[k]


@contextlib.contextmanager
def poisoned(pattern):
  """Run the body with the strict workspace and poisoned device allocations of `pattern`; check every guard band
  on exit."""
  from dynibar_b200 import render_ray
  p = Poison(pattern)
  render_ray.new_frame()  # the packed source views of an earlier frame live in memory poisoned with another pattern
  with pytest.MonkeyPatch.context() as mp:
    mp.setattr(_lib, "workspace", p)
    mp.setattr(torch, "empty", p.empty)
    mp.setattr(torch, "empty_like", p.empty_like)
    yield p
    p.check()
  render_ray.new_frame()


# ---- collecting and comparing what a scenario returns ----
def flatten(obj, prefix="", out=None):
  """{path: detached CPU copy} of every tensor in nested dicts / lists / tuples (numpy arrays become tensors)."""
  import numpy as np
  out = {} if out is None else out
  if torch.is_tensor(obj):
    out[prefix] = obj.detach().cpu().clone()
  elif isinstance(obj, np.ndarray):
    out[prefix] = torch.from_numpy(obj.copy())
  elif isinstance(obj, dict):
    for k, v in obj.items():
      flatten(v, "%s/%s" % (prefix, k), out)
  elif isinstance(obj, (list, tuple)):
    for i, v in enumerate(obj):
      flatten(v, "%s[%d]" % (prefix, i), out)
  return out


def bits(t):
  t = t.contiguous().reshape(-1)
  return t.view(torch.uint8) if t.numel() else t


def assert_bit_identical(runs, what):
  """runs: {label: flat dict}, the first one the base.  Every tensor equal bit for bit (NaN payloads included) to the
  base run's."""
  (base_label, base), = list(runs.items())[:1]
  assert base, "%s: the scenario returned no tensors" % what
  for label, got in runs.items():
    assert sorted(got) == sorted(base), (what, label)
    for k, v in base.items():
      g = got[k]
      assert g.shape == v.shape and g.dtype == v.dtype, (what, label, k)
      if not torch.equal(bits(g), bits(v)):
        d = (g.double() - v.double()).abs()
        raise AssertionError("%s: %s of run %s differs from run %s in %d of %d elements (max |diff| %s, %d non-finite)"
                             % (what, k, label, base_label, int((bits(g) != bits(v)).sum()), v.numel(),
                                d.max().item() if d.numel() else 0, int((~torch.isfinite(g.double())).sum())))
