"""The workspace and scratch sizes the library declares grow with the problem: every dyn_*_workspace_bytes /
*_scratch_bytes function is non-decreasing in each of its shape arguments over a grid of shapes across the kernels'
tile and threshold edges.  A size that shrinks as a shape grows is a sizing formula that forgot a term somewhere,
and a caller that sizes a shared buffer for its largest call would then hand a later call too little.

The nets' sizes hold one internal chunk of rays (net_rows_per_chunk = 4 Mi rows / (S V)), so along S and V they are
compared where the rays fit one chunk at both shapes; along R they are compared everywhere.  The sizes computed with
the device (the splatting's radix-sort scratch) are left to tests/test_memory_contract_gpu.py."""

import itertools

import pytest

from dynibar_b200 import _lib

L = _lib.lib
CHUNK_ROWS = 4 << 20
RS = (1, 2, 37, 63, 64, 65, 127, 128, 129, 255, 256, 257, 2047, 2048, 2049, 4097, 8192)
SS = (1, 2, 5, 16, 20, 32, 63, 64, 65, 127, 128, 129, 191, 192, 193, 256, 384)
VS = (1, 2, 7, 8, 9, 15, 16, 17, 31, 32)


def _along(grid, axis):
  """Pairs of grid points that differ in one coordinate, `axis`, by one step of its list."""
  for point in itertools.product(*grid):
    i = grid[axis].index(point[axis])
    if i + 1 < len(grid[axis]):
      yield point, point[:axis] + (grid[axis][i + 1],) + point[axis + 1:]


def _check(fn, grid, keep=lambda a, b: True):
  bad = []
  for axis in range(len(grid)):
    for a, b in _along(grid, axis):
      if keep(a, b) and fn(*b) < fn(*a):
        bad.append((a, fn(*a), b, fn(*b)))
  assert not bad, "%d decreasing steps, e.g. %s" % (len(bad), bad[:4])


def _one_chunk(a, b):
  """(R, S, V) pairs: every step along R, steps along S or V where the rays fit one chunk at both ends."""
  return a[1:] == b[1:] or max(a[0] * a[1] * a[2], b[0] * b[1] * b[2]) <= CHUNK_ROWS


@pytest.mark.parametrize("name", ["dyn_net_workspace_bytes", "dyn_net_fused_workspace_bytes",
                                  "dyn_net_train_workspace_bytes", "dyn_net_backward_scratch_bytes"])
@pytest.mark.parametrize("kind", [_lib.NET_DYNAMIC, _lib.NET_STATIC])
def test_net_sizes_grow(name, kind):
  fn = getattr(L, name)
  _check(lambda R, S, V: fn(kind, R, S, V), (RS, SS, VS), _one_chunk)


def test_motion_sizes_grow():
  _check(L.dyn_motion_workspace_bytes, (RS, SS))
  _check(L.dyn_motion_train_workspace_bytes, (RS + (65573, 131072),))


def test_criterion_size_grows():
  _check(L.dyn_mono_loss_workspace_bytes, (tuple(sorted(set(range(1, 70)) | set(RS) | {3072, 65536})),))


@pytest.mark.parametrize("name", ["dyn_encoder_workspace_bytes", "dyn_encoder_train_workspace_bytes",
                                  "dyn_encoder_backward_scratch_bytes"])
def test_encoder_sizes_grow(name):
  sizes = (8, 16, 17, 33, 64, 72, 90, 96, 128, 150, 206, 288, 354)
  _check(getattr(L, name), ((1, 2, 3, 8), sizes, sizes))


def test_scoring_scene_and_trajectory_sizes_grow():
  _check(L.dyn_image_scores_workspace_bytes, ((1, 3, 11, 16, 17), (8, 37, 45, 64, 288), (9, 56, 71, 512)))
  _check(L.dyn_scene_masks_workspace_bytes, ((1, 3, 24), (1, 20, 37, 288), (1, 30, 71, 512)))
  _check(L.dyn_traj_combine_grad_d_workspace_bytes, ((1, 6, 7), (1, 4, 8), (1, 255, 256, 257, 4096, 65537)))
