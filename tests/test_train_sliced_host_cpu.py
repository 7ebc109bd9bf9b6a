"""The slice plan of a sliced training step (dynibar_b200.train_step.slice_plan), on the host."""

import pytest

from dynibar_b200 import train_step as ts


def _check(R, slice_rays, S):
  spans = ts.slice_plan(R, slice_rays, S)
  # the slices cover the batch in order, without gap or overlap
  assert spans[0][0] == 0 and spans[-1][1] == R
  assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
  assert all(0 < hi - lo <= max(slice_rays, R if len(spans) == 1 else 0) for lo, hi in spans)
  # every slice starts on a multiple of 8 rays; only the last may hold a count that is not one
  assert all(lo % 8 == 0 for lo, _ in spans)
  assert all((hi - lo) % 8 == 0 for lo, hi in spans[:-1])
  # near-equal: the last slice is at most 8 rays per slice short of the others
  sizes = [hi - lo for lo, hi in spans]
  assert max(sizes) - min(sizes) < 8 * len(spans)
  # every slice on the batch's side of each row-count threshold (tests/train_step_ref._check_chunk), except that a
  # batch of 2048 rays or more may run slices below 2048 rays, all of them
  for lo, hi in spans:
    n = hi - lo
    assert (R >= 128) == (n >= 128)
    for lim in (128, 2048):
      assert (R * S >= lim) == (n * S >= lim)
  assert len({(hi - lo) >= 2048 for lo, hi in spans}) == 1
  return spans


@pytest.mark.parametrize("R,slice_rays,S", [
    (1024, 1024, 64), (1024, 2048, 64), (3072, 3072, 64), (96, 128, 64),  # a batch that fits is one slice
    (3072, 1024, 64), (1024, 512, 64), (1000, 512, 64), (1024, 384, 64), (1000, 384, 64), (105, 64, 64),
    (105, 56, 64), (4096, 2048, 64), (4090, 2048, 64), (2500, 1000, 32), (700, 256, 2), (20000, 1024, 64)])
def test_slice_plan_covers_the_batch(R, slice_rays, S):
  spans = _check(R, slice_rays, S)
  if R <= slice_rays:
    assert spans == [(0, R)]


def test_slice_plan_shapes():
  assert ts.slice_plan(3072, 1024, 64) == [(0, 1024), (1024, 2048), (2048, 3072)]
  assert ts.slice_plan(1024, 512, 64) == [(0, 512), (512, 1024)]
  assert ts.slice_plan(1000, 512, 64) == [(0, 504), (504, 1000)]
  assert ts.slice_plan(1024, 384, 64) == [(0, 344), (344, 688), (688, 1024)]
  # 4090 rays in two slices of at most 2048 would put one on each side of 2048 rays: three slices below it
  assert [hi - lo for lo, hi in ts.slice_plan(4090, 2048, 64)] == [1368, 1368, 1354]


@pytest.mark.parametrize("R,slice_rays,S", [
    (136, 128, 64),    # two slices of <= 128 rays: one would fall below the 128-ray forward threshold
    (256, 100, 64),    # any slice of <= 100 rays falls below it, the batch does not
    (64, 16, 64),      # 16 rays x 64 samples = 1024 rows, below the 2048-row backward threshold; the batch is not
    (105, 40, 64),     # 40 + 40 + 25 rays or 4 x <= 32: a last slice below 32 rays x 64 samples = 2048 rows
    (100, 4, 64),      # no slice of at most 4 rays starts every slice on a multiple of 8
    (0, 128, 64), (128, 0, 64)])
def test_slice_plan_refuses(R, slice_rays, S):
  with pytest.raises(ValueError):
    ts.slice_plan(R, slice_rays, S)
