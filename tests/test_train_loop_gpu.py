"""The monocular training loop (dynibar_b200.trainer.Trainer) on the device, on a small synthetic scene
(tests/mono_scene_ref.write_scene: 8 frames of 48 x 64, 512 rays in 256-ray slices, 32 samples, bf16).

  1. The loop against the same steps written out by hand from MonocularScene.sample, mono_step_backward and Adam,
     across the warm-up / main boundary: batches, epochs and per-group learning rates bit for bit; parameters within
     2x the spread of two identical hand runs (relative L2 per optimiser group, SPREAD_BARS; the network backward's
     float atomics make runs differ in the last bits, and Adam carries that forward).
  2. Resume: k steps, save, a new Trainer from the file, m more steps, against k + m uninterrupted steps (inside the
     warm-up, and in the main phase): the same data stream, epochs, learning rates, scheduler state and Adam step counts;
     parameters within the same bar.
  3. save -> load -> save gives identical tensors.
  4. The checkpoint renders through tools/render_monocular_bt.py's loading path, as the trainer's own model does.
  5. Under torch.cuda.set_sync_debug_mode("warn"): a loop step that neither logs, saves nor renders synchronises no
     more often than the bare hand-written step, and a print step adds only its read-back.
"""

import copy
import os
import tempfile
import warnings
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import mono_scene_ref as msr
from dynibar_b200 import model as dmodel, sample_ray, trainer as tr, train_step as ts
from dynibar_b200.feature_network import ResNet
from dynibar_b200.projection import Projector

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
N, H, W = 8, 48, 64
BIG = 10 ** 9


def _args(**kw):
  a = dict(training_height=H, num_source_views=3, max_range=9, num_vv=3, mask_src_view=True, erosion_radius=3,
           N_rand=512, slice_rays=256, sample_mode="uniform", N_samples=32, inv_uniform=True, det=False,
           init_decay_epoch=2, n_iters=BIG, i_print=BIG, i_img=BIG, i_weights=BIG, chunk_size=4096,
           coarse_feat_dim=32, fine_feat_dim=32, num_basis=6, anti_alias_pooling=1, mask_rgb=1, input_dir=True,
           input_xyz=False, occ_weights_mode=0, lrate_mlp=4e-4, lrate_feature=8e-4, lrate_decay_factor=0.5,
           w_disp=0.1, w_flow=0.01, w_cycle=0.1, cycle_factor=0.1, anneal_cycle=True, w_reg=0.05,
           w_skew_entropy=5e-4, w_distortion=1e-3, decay_rate=10.0, ckpt_path="", pretrain_path="", no_reload=False,
           expname="t", rootdir=".")
  a.update(kw)
  return SimpleNamespace(**a)


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
  from dynibar_b200 import mono_scene
  root = tmp_path_factory.mktemp("train_loop")
  path = msr.write_scene(str(root / "s" / "dense"), msr.synthetic_scene(21, N, H, W, mask_hw=(40, 70)))
  return mono_scene.MonocularScene(path, _args(), DEV)


def _seed():
  torch.manual_seed(7)
  sample_ray.rng = np.random.RandomState(234)


class Recording(tr.Trainer):
  """A Trainer that records each step's batch, epoch, phase and the groups' learning rates after it."""

  def __init__(self, *a, **kw):
    # global step 0 of a main phase prints, saves and renders (0 % i == 0, as in train.py)
    kw.setdefault("out_folder", tempfile.mkdtemp())
    super().__init__(*a, log=lambda s: None, **kw)
    self.record = []

  def step(self, train_data, rb, epoch, bootstrap, sched_step):
    out = super().step(train_data, rb, epoch, bootstrap, sched_step)
    self.record.append(_entry(train_data, rb, epoch, bootstrap, self.optimizer))
    return out


def _entry(td, rb, epoch, bootstrap, opt):
  return dict(epoch=epoch, bootstrap=bootstrap, lrs=[g["lr"] for g in opt.param_groups],
              sel=np.asarray(rb["selected_inds"]).copy(), ids=(int(td["id"]), int(td["anchor_id"])),
              rays=torch.cat([rb["ray_o"], rb["ray_d"], rb["rgb"]], 1).clone(),
              views=torch.cat([rb["src_rgbs"].flatten(), rb["static_src_rgbs"].flatten()]).clone())


def _fresh(scene, args, **kw):
  _seed()
  return Recording(args, scene, DEV, **kw)


def hand_run(scene, args, init, schedule):
  """`schedule`: [(phase, epoch, sched_step)] written out by hand; the step of train.py:116-199 / :227-470 from
  scene.sample, the encoders, mono_step_backward and a six-group Adam built here."""
  _seed()
  m = tr.build_model(args, N, DEV)
  for k in tr.NETS:
    getattr(m, k).load_state_dict(init[k])
  with torch.no_grad():
    m.trajectory_basis.copy_(init["traj_basis"])
  lm, lf = args.lrate_mlp, args.lrate_feature
  opt = torch.optim.Adam([{"params": m.net_coarse_st.parameters(), "lr": lm * 0.5},
                          {"params": m.feature_net_st.parameters(), "lr": lf * 0.5},
                          {"params": m.net_coarse_dy.parameters(), "lr": lm},
                          {"params": m.feature_net.parameters(), "lr": lf},
                          {"params": m.motion_mlp.parameters(), "lr": lm},
                          {"params": m.trajectory_basis, "lr": lm * 0.25}])
  sched = torch.optim.lr_scheduler.StepLR(opt, step_size=N * args.init_decay_epoch, gamma=args.lrate_decay_factor)
  rng = np.random.RandomState(0)
  proj = Projector(DEV)
  record = []
  for phase, epoch, sched_step in schedule:
    scene.set_epoch(epoch)
    td, rb = scene.sample(rng, args.N_rand, args.sample_mode)
    hand_step(td, rb, m, opt, sched, proj, args, epoch, phase == "warmup", sched_step)
    record.append(_entry(td, rb, epoch, phase == "warmup", opt))
  return m, opt, sched, record


def hand_step(td, rb, m, opt, sched, proj, args, epoch, bootstrap, sched_step):
  i, an = int(td["id"]), int(td["anchor_id"])
  offs = ([int(j) - i for j in td["nearest_pose_ids"][0]], [int(j) - an for j in td["anchor_nearest_pose_ids"][0]])
  fm = (m.feature_net(rb["src_rgbs"][0].permute(0, 3, 1, 2).contiguous())[0],
        m.feature_net(rb["anchor_src_rgbs"][0].permute(0, 3, 1, 2).contiguous())[0],
        m.feature_net_st(rb["static_src_rgbs"][0].permute(0, 3, 1, 2).contiguous())[0])
  opt.zero_grad()
  ts.mono_step_backward((i, an), (td["ref_time"], td["anchor_time"]), offs, rb, m, fm, proj, args.N_samples, args,
                        epoch, slice_rays=args.slice_rays, bootstrap=bootstrap, inv_uniform=args.inv_uniform,
                        det=args.det, num_vv=args.num_vv)
  opt.step()
  if sched_step:
    sched.step()


def _init_state(t):
  st = {k: copy.deepcopy(getattr(t.model, k).state_dict()) for k in tr.NETS}
  st["traj_basis"] = t.model.trajectory_basis.detach().clone()
  return st


def _groups(opt):
  return [torch.cat([p.detach().flatten() for p in g["params"]]) for g in opt.param_groups]


def _rel(a, b):
  return [((x - y).norm() / y.norm().clamp_min(1e-30)).item() for x, y in zip(a, b)]


def _same_stream(got, want):
  assert len(got) == len(want)
  for k, (g, w) in enumerate(zip(got, want)):
    assert g["epoch"] == w["epoch"] and g["bootstrap"] == w["bootstrap"] and g["ids"] == w["ids"], k
    assert g["lrs"] == w["lrs"], (k, g["lrs"], w["lrs"])
    assert np.array_equal(g["sel"], w["sel"]), k
    assert torch.equal(g["rays"], w["rays"]) and torch.equal(g["views"], w["views"]), k


# relative L2 per optimiser group: 2x the largest spread of two identical runs measured over five calls of tests 1 and
# 2 on an H100 80GB HBM3 (700 W power limit).  One pair's spread varies up to 10x from call to call (motion_mlp
# 2.8e-5 .. 2.9e-4), so each test's own pair only widens the bar.
SPREAD_BARS = {"net_coarse_st": 2.4e-4, "feature_net_st": 9e-4, "net_coarse_dy": 2.7e-4, "feature_net": 1.3e-3,
               "motion_mlp": 6e-4, "trajectory_basis": 1.7e-4}


def _within_spread(got, ref, ref2, what):
  spread, err = _rel(ref2, ref), _rel(got, ref)
  names = [g[0] for g in tr.GROUPS]
  for n, s, e in zip(names, spread, err):
    print("  %s %-15s spread %.3e  difference %.3e" % (what, n, s, e))
  bad = [(n, e, s) for n, s, e in zip(names, spread, err) if not e <= max(2.0 * s, SPREAD_BARS[n])]
  assert not bad, bad


def test_loop_matches_the_hand_written_steps(scene):
  args = _args(init_decay_epoch=2)  # the warm-up is epoch 0 (8 steps); then main epoch 0
  steps = N + 3
  t = _fresh(scene, args)
  init = _init_state(t)
  assert t.run(steps) == steps
  schedule = [("warmup", 0, False)] * N + [("main", 0, True)] * 3
  assert [(r["bootstrap"], r["epoch"]) for r in t.record] == [(p == "warmup", e) for p, e, _ in schedule]
  _, opt1, sched1, rec1 = hand_run(scene, args, init, schedule)
  _, opt2, _, _ = hand_run(scene, args, init, schedule)
  _same_stream(t.record, rec1)
  assert t.scheduler.state_dict() == sched1.state_dict() and t.global_step == N + 3
  _within_spread(_groups(t.optimizer), _groups(opt1), _groups(opt2), "loop-vs-hand")


@pytest.mark.parametrize("ide,k,m", [(4, N, 4), (1, N, 3)], ids=["in_warmup", "main"])
def test_resume_continues_the_run(scene, tmp_path, ide, k, m):
  args = _args(init_decay_epoch=ide)
  whole = []
  for _ in range(2):  # one after the other: each run starts from the seeded generators
    whole.append(_fresh(scene, args))
    whole[-1].run(k + m)
  first = _fresh(scene, args)
  first.run(k)
  path = str(tmp_path / "model_latest.pth")
  first.save(path, first.global_step)
  assert first.global_step == k
  second = Recording(_args(init_decay_epoch=ide, ckpt_path=path), scene, DEV)
  assert second.start_step == k
  second.run(m)
  _same_stream(first.record + second.record, whole[0].record)
  assert second.scheduler.state_dict() == whole[0].scheduler.state_dict()
  assert second.global_step == whole[0].global_step
  counts = set()
  for g1, g2 in zip(second.optimizer.param_groups, whole[0].optimizer.param_groups):
    for p1, p2 in zip(g1["params"], g2["params"]):
      s1, s2 = second.optimizer.state.get(p1), whole[0].optimizer.state.get(p2)
      assert (s1 is None) == (s2 is None)  # tensors no step has a gradient for (the warm-up's dynamic nets)
      if s1 is not None:
        assert int(s1["step"]) == int(s2["step"])
        counts.add(int(s1["step"]))
  assert k + m in counts
  _within_spread(_groups(second.optimizer), _groups(whole[0].optimizer), _groups(whole[1].optimizer),
                 "resumed-vs-whole")


def _tensors(x, prefix=""):
  if torch.is_tensor(x):
    return {prefix: x}
  if isinstance(x, dict):
    out = {}
    for k, v in x.items():
      out.update(_tensors(v, "%s/%s" % (prefix, k)))
    return out
  if isinstance(x, (list, tuple)):
    out = {}
    for i, v in enumerate(x):
      out.update(_tensors(v, "%s/%d" % (prefix, i)))
    return out
  return {prefix: x}


def test_save_load_save_round_trip(scene, tmp_path):
  args = _args(init_decay_epoch=1)
  t = _fresh(scene, args)
  t.run(2)
  a, b = str(tmp_path / "a_latest.pth"), str(tmp_path / "b.pth")
  t.save(a, t.global_step)
  u = Recording(_args(init_decay_epoch=1, ckpt_path=a), scene, DEV)
  u.save(b, u.start_step)
  ta = _tensors(torch.load(a, map_location="cpu", weights_only=False))
  tb = _tensors(torch.load(b, map_location="cpu", weights_only=False))
  assert sorted(ta) == sorted(tb)
  for k in ta:
    if torch.is_tensor(ta[k]):
      assert ta[k].dtype == tb[k].dtype and torch.equal(ta[k], tb[k]), k
    elif isinstance(ta[k], np.ndarray):
      assert np.array_equal(ta[k], tb[k]), k
    else:
      assert ta[k] == tb[k], k


def test_checkpoint_renders_through_the_render_tool_loader(scene, tmp_path):
  from dynibar_b200.render_image import render_single_image_mono
  args = _args(init_decay_epoch=1)
  t = _fresh(scene, args)
  t.run(2)
  path = str(tmp_path / "model_latest.pth")
  t.save(path, t.global_step)
  # tools/render_monocular_bt.py's loading path
  model, info = dmodel.model_from_checkpoints(args, coarse=path, mono=True, device=DEV)
  for k in ("feature_net", "feature_net_st"):
    enc = ResNet().to(DEV)
    enc.load_state_dict(dmodel._strip(info["encoders"][k]))
    setattr(model, k, enc.eval().requires_grad_(False))
  assert info["coarse_step"] == 2
  scene.set_epoch(0)
  td, _ = scene.sample(np.random.RandomState(3), 64, "uniform")
  frame, tm, offs = t.batch(td)

  def render(m):
    with torch.no_grad():
      rb = scene.get_all(td)
      fm = (m.feature_net(rb["src_rgbs"][0].permute(0, 3, 1, 2).contiguous())[0], None,
            m.feature_net_st(rb["static_src_rgbs"][0].permute(0, 3, 1, 2).contiguous())[0])
      return render_single_image_mono(frame, tm, offs, SimpleNamespace(H=H, W=W), rb, m, Projector(DEV), 4096,
                                      args.N_samples, args, inv_uniform=True, det=True, featmaps=fm, is_train=False,
                                      num_vv=args.num_vv)["outputs_coarse_ref"]["rgb"]

  got, want = render(model), render(t.model)
  assert got.shape == (H, W, 3) and torch.isfinite(got).all()
  assert torch.equal(got, want)
  # and the trainer's own training-view PNGs
  t.out_folder = str(tmp_path)
  d = t.render_view(td, 2)
  assert sorted(os.listdir(d)) == sorted(n + ".png" for n in (
      "render_rgb_coarse_ref", "render_rgb_coarse_anchor", "render_rgb_static", "render_rgb_dynamic", "st_rgb_pred",
      "gt_rgb_coarse", "render_depth_coarse", "occ_weight_map"))


def _syncs(fn):
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode("warn")
  try:
    with warnings.catch_warnings(record=True) as w:
      warnings.simplefilter("always")
      fn()
  finally:
    torch.cuda.set_sync_debug_mode(0)
  torch.cuda.synchronize()
  return sum("synchroniz" in str(x.message) for x in w)


def test_loop_adds_no_synchronisation(scene):
  args = _args(init_decay_epoch=1, i_print=3)
  _seed()
  t = tr.Trainer(args, scene, DEV, out_folder=tempfile.mkdtemp(), log=lambda s: None)  # records nothing
  t.run(1)  # global step 0 printed; warm every shape
  m, opt, sched = t.model, t.optimizer, t.scheduler

  def pair():
    """(syncs of a bare hand-written step, syncs of the loop's next step), both on the batch the loop draws next: the
    ids the step reads back vary in number with the draw."""
    rng, pixels = np.random.RandomState(), sample_ray.rng.get_state()
    rng.set_state(t.rng.get_state())

    def bare():
      td, rb = scene.sample(rng, args.N_rand, args.sample_mode)
      hand_step(td, rb, m, opt, sched, t.projector, args, 0, False, True)

    hand = _syncs(bare)
    sample_ray.rng.set_state(pixels)
    return hand, _syncs(lambda: t.run(1))

  hand, quiet = pair()      # global step 1
  pair()                    # global step 2
  hand3, printed = pair()   # global step 3: prints
  print("\nsynchronisations per step: bare hand-written %d, loop %d; bare hand-written %d, loop with print %d"
        % (hand, quiet, hand3, printed))
  assert hand > 0
  assert quiet <= hand
  assert printed <= hand3 + 1
