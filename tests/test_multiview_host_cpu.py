"""Host logic of multi-camera ray batches (no GPU): stacking K target cameras' batches of one time step,
splitting the rendered outputs back per camera, sharding the stacked rays over ranks, and the argument checks
of the multi-camera C-ABI entry points, which run before any CUDA call."""

import os
import socket
from collections import OrderedDict

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import scenes
from dynibar_b200 import distributed as dd
from dynibar_b200 import sample_ray as sr
from dynibar_b200 import synthetic

H, W = 12, 16


def _batches(K=3, seed=31):
  batch, _, _, _, _, _ = synthetic.make_scene(H=H, W=W, V_dy=7, V_st=5, seed=seed)
  data = scenes.sampler_data(batch, H, W, seed)
  K_mat = sr.parse_camera(batch["camera"])[2][0]
  out = []
  for k in range(K):
    c2w = torch.eye(4)
    c2w[0, 3] = 0.03 * k
    smp = sr.RaySamplerSingleImage(dict(data, camera=synthetic.camera_vector(H, W, K_mat, c2w)[None]), "cpu")
    out.append(smp.get_all())
  return out


def test_stack_ray_batches_round_trips():
  parts = _batches()
  batch, counts, hw = sr.stack_ray_batches(parts)
  assert counts == [H * W] * 3 and hw == (H, W)
  assert batch["camera"].shape == (3, 34)
  assert batch["camera_index"].dtype == torch.int32
  assert batch["camera_index"].tolist() == [k for k in range(3) for _ in range(H * W)]
  for k in ("src_cameras", "static_src_cameras", "depth_range", "src_rgbs", "static_src_rgbs"):
    assert batch[k] is parts[0][k]  # per-frame tensors are shared, not copied
  for k in ("ray_o", "ray_d", "uv_grid", "rgb", "disp", "motion_mask", "static_mask", "camera"):
    for p, piece in zip(parts, batch[k].split(counts if k != "camera" else 1, 0)):
      assert torch.equal(piece, p[k]), k
  for k in ("flows", "masks"):
    for p, piece in zip(parts, batch[k].split(counts, 1)):
      assert torch.equal(piece, p[k]), k
  # one camera: the batch is today's, plus an all-zero index
  one, counts1, _ = sr.stack_ray_batches(parts[:1])
  assert counts1 == [H * W] and one["camera"].shape == (1, 34) and not one["camera_index"].any()


@pytest.mark.parametrize("key", ["src_cameras", "static_src_cameras", "depth_range", "src_rgbs",
                                 "static_src_rgbs"])
def test_stack_ray_batches_rejects_batches_of_other_time_steps(key):
  parts = _batches()
  other = parts[2][key].clone()
  other.view(-1)[0] += 0.5
  parts[2] = dict(parts[2], **{key: other})
  with pytest.raises(ValueError, match=key):
    sr.stack_ray_batches(parts)
  # equal values in another tensor are accepted
  parts = _batches()
  parts[1] = dict(parts[1], **{key: parts[1][key].clone()})
  sr.stack_ray_batches(parts)


def test_stack_ray_batches_rejects_more_than_16_cameras():
  parts = _batches(K=1)
  with pytest.raises(ValueError, match="1..16"):
    sr.stack_ray_batches(parts * 17)


def test_per_camera_split_matches_single_camera_merge():
  from dynibar_b200.render_image import _merge, _merge_multi
  g = torch.Generator().manual_seed(4)
  hws = [(3, 5), (3, 5), (2, 7)]
  counts = [h * w for h, w in hws]
  S = 6

  def outputs(n):
    return OrderedDict([("rgb", torch.rand(n, 3, generator=g)), ("depth", torch.rand(n, generator=g)),
                        ("weights", torch.rand(n, S, generator=g)), ("mask", torch.rand(n, generator=g) > 0.3),
                        ("render_flows", torch.rand(4, n, 2, generator=g))])

  per_cam = [outputs(n) for n in counts]
  full = OrderedDict((k, torch.cat([p[k] for p in per_cam], 1 if k == "render_flows" else 0)) for k in per_cam[0])
  # chunks of 8 rays straddle every camera boundary (15, 30)
  chunks = [OrderedDict((k, v[:, i:i + 8] if k == "render_flows" else v[i:i + 8]) for k, v in full.items())
            for i in range(0, sum(counts), 8)]
  got = _merge_multi(chunks, counts, hws)
  assert len(got) == 3
  for g_k, p, (h, w) in zip(got, per_cam, hws):
    want = _merge([p], h, w)
    assert list(g_k.keys()) == list(want.keys())
    for k in want:
      assert g_k[k].shape == want[k].shape and g_k[k].dtype == want[k].dtype, k
      assert torch.equal(g_k[k], want[k]), k
  assert _merge_multi([], counts, hws) == [OrderedDict()] * 3


def _free_port():
  s = socket.socket()
  s.bind(("127.0.0.1", 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _render_stub(batch):
  # per-ray function of the ray and of its target camera
  o, d = batch["ray_o"], batch["ray_d"]
  c = batch["camera"][batch["camera_index"].long()][:, 18:34]
  return torch.cat([torch.sin(o + 2 * d), (c * c).sum(-1, keepdim=True) * d[:, :1],
                    batch["camera_index"][:, None].float()], 1)


def _shard_worker(rank, world, port, q):
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  batch, counts, _ = sr.stack_ray_batches(_batches())
  local, (lo, hi) = dd.shard_ray_batch(batch, rank, world)
  assert local["camera_index"].shape[0] == local["ray_o"].shape[0] == hi - lo
  assert torch.equal(local["camera_index"], batch["camera_index"][lo:hi])
  assert torch.equal(local["ray_o"], batch["ray_o"][lo:hi])
  assert local["camera"] is batch["camera"]
  frame = dd.render_frame_sharded(_render_stub, batch)
  if rank == 0:
    q.put(torch.equal(frame, _render_stub(batch)) and [int(n) for n in
                                                        torch.bincount(frame[:, -1].long())] == counts)
  else:
    assert frame is None
  dist.barrier()
  dist.destroy_process_group()


def test_two_rank_sharding_slices_camera_index_with_the_rays():
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  port = _free_port()
  procs = [ctx.Process(target=_shard_worker, args=(r, 2, port, q)) for r in range(2)]
  for p in procs:
    p.start()
  ok = q.get(timeout=120)
  for p in procs:
    p.join(timeout=120)
    assert p.exitcode == 0
  assert ok


@pytest.mark.parametrize("K,with_index,msg", [(17, True, b"K = 17"), (0, True, b"K = 0"),
                                              (3, False, b"per-ray camera index")])
def test_multi_camera_entry_points_check_arguments_before_any_cuda_call(K, with_index, msg):
  from dynibar_b200 import _lib
  lib = _lib.lib
  fake = 0x1000  # never dereferenced: the checks return first
  idx = fake if with_index else None
  R, S, V = 8, 16, 5
  rc = lib.dyn_net_static_fused_mc(None, fake, fake, fake, fake, K, idx, fake, fake, fake, R, S, V, H, W, 32,
                                   H // 4, W // 4, fake, fake, fake, 1 << 20, None)
  assert rc == -1 and msg in lib.dyn_last_error()
  rc = lib.dyn_project_gather_mc(fake, None, fake, K, idx, fake, fake, fake, V, R, S, H, W, 32, H // 4, W // 4,
                                 fake, fake, fake, fake, None)
  assert rc == -1 and msg in lib.dyn_last_error()
