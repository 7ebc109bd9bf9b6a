"""The monocular training loop's host side (dynibar_b200.trainer, tools/train.py) without a GPU.

  1. `plan` against a literal restatement of train.py:111-573's control flow that steps a real torch StepLR: a fresh
     start crossing from the warm-up to the main phase, a resume inside the warm-up, a resume past it, the n_iters
     stop, the model_no-vv trigger and the 5e-7 lr floor; and two planted errors (the scheduler stepping in the
     warm-up, the main phase's epoch continuing after the warm-up) that the comparison must catch.
  2. tools/train.py's config parser on the shipped train_kid-running.txt, with command-line overrides.
  3. The optimiser's six groups, their order and initial learning rates.
  4. A checkpoint made on the CPU: the reference's keys plus the RNG key, loadable by model_from_checkpoints(mono=True),
     its optimizer state loadable into a fresh six-group Adam, and the loop's RNG restored from it.
"""

import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dynibar_b200 import model as dmodel, sample_ray, trainer as tr

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import train as train_tool  # noqa: E402

# the restatement steps a StepLR whose optimiser never steps
pytestmark = pytest.mark.filterwarnings("ignore:Detected call of `lr_scheduler.step\\(\\)` before")


# ---------------------------------------------------------------------------------------------------------------
# 1. the plan
# ---------------------------------------------------------------------------------------------------------------
def literal(num_frames, n_iters, init_decay_epoch, start_step, i_print, i_img, i_weights, lrate, gamma,
            sched_steps=0, sched_in_warmup=False, continue_epoch=False):
  """train.py:111-573 written out with a real Adam / StepLR on one parameter; `sched_steps` scheduler steps (with the
  floor test) taken before the loop, as a resumed checkpoint's scheduler would have.  The two flags plant errors."""
  p = torch.nn.Parameter(torch.zeros(1))
  opt = torch.optim.Adam([{"params": [p], "lr": lrate}])
  sched = torch.optim.lr_scheduler.StepLR(opt, step_size=num_frames * init_decay_epoch, gamma=gamma)
  for _ in range(sched_steps):
    if sched.get_last_lr()[0] > 5e-7:
      sched.step()
  lr0, ep0 = sched.get_last_lr()[0], sched.last_epoch
  out, files = [], set()
  global_step = start_step
  start_epoch = global_step // num_frames
  for epoch in range(start_epoch, init_decay_epoch // 2):
    for ii in range(num_frames):
      stepped = False
      if sched_in_warmup and sched.get_last_lr()[0] > 5e-7:
        sched.step()
        stepped = True
      global_step += 1
      acts = []
      if global_step % i_img == 0:
        acts.append("render")
      out.append(("warmup", epoch, global_step, stepped, sched.get_last_lr()[0], tuple(acts)))
  first_main = init_decay_epoch // 2 if continue_epoch else start_epoch
  for epoch in range(first_main, int(10 ** 5)):
    if global_step > start_step + n_iters + 1:
      break
    for ii in range(num_frames):
      stepped = False
      if sched.get_last_lr()[0] > 5e-7:
        sched.step()
        stepped = True
      acts = []
      if epoch + 1 == init_decay_epoch * 5:
        if "model_no-vv.pth" not in files:
          files.add("model_no-vv.pth")
          acts.append("save_no_vv")
      if global_step % i_print == 0:
        acts.append("print")
      if global_step % i_weights == 0:
        acts.append("save_latest")
      if global_step % i_img == 0:
        acts.append("render")
      out.append(("main", epoch, global_step, stepped, sched.get_last_lr()[0], tuple(acts)))
      global_step += 1
  return out, (lr0, ep0, num_frames * init_decay_epoch)


def planned(num_frames, n_iters, init_decay_epoch, start_step, i_print, i_img, i_weights, lrate, gamma,
            sched_steps=0):
  """tr.plan from the scheduler state `literal` starts from."""
  _, (lr0, ep0, step_size) = literal(num_frames, -10 ** 6, init_decay_epoch, 0, 1, 1, 1, lrate, gamma, sched_steps)
  return [tuple(s) for s in tr.plan(num_frames, n_iters, init_decay_epoch, start_step, i_print, i_img, i_weights,
                                    lr0, step_size, gamma, ep0)]


CASES = {  # num_frames, n_iters, init_decay_epoch, start_step, i_print, i_img, i_weights, lrate, gamma, sched_steps
    "fresh_crosses_warmup": (5, 30, 4, 0, 3, 4, 7, 2e-4, 0.5, 0),
    "resume_in_warmup": (5, 30, 4, 7, 3, 4, 7, 2e-4, 0.5, 0),
    "resume_past_warmup": (5, 30, 4, 23, 3, 4, 7, 2e-4, 0.5, 13),
    "n_iters_stop_mid_epoch": (6, 9, 2, 0, 2, 5, 4, 2e-4, 0.5, 0),
    "no_vv_trigger": (3, 20, 1, 0, 4, 100, 100, 2e-4, 0.5, 0),
    "no_vv_trigger_on_resume": (3, 20, 1, 13, 4, 100, 100, 2e-4, 0.5, 13),
    "lr_floor": (4, 60, 1, 0, 5, 100, 9, 4e-6, 0.5, 0),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_plan_restates_train_py(case):
  c = CASES[case]
  want, _ = literal(*c)
  got = planned(*c)
  assert got == want
  phases = [s[0] for s in got]
  if case == "fresh_crosses_warmup":
    assert phases.count("warmup") == 2 * 5 and "main" in phases
    main = [s for s in got if s[0] == "main"]
    assert main[0][1] == 0 and main[0][2] == 10  # the epoch restarts; the step count does not
  if case == "resume_in_warmup":
    assert got[0][:3] == ("warmup", 1, 8)
  if case == "resume_past_warmup":
    assert "warmup" not in phases and got[0][1] == 4
  if case == "n_iters_stop_mid_epoch":  # the stop test runs only at the start of an epoch
    assert got[-1][2] == 11 and len(got) % 6 == 0 and got[-1][2] > 9 + 1 - 6
  if case.startswith("no_vv"):
    assert sum("save_no_vv" in s[5] for s in got) == 1
    assert [s for s in got if "save_no_vv" in s[5]][0][1] == 4
  if case == "lr_floor":
    stepped = [s[3] for s in got]
    assert stepped[0] and not stepped[-1]
    assert min(s[4] for s in got) <= 5e-7 < max(s[4] for s in got)
    # once at or below the floor the scheduler never steps again
    first_off = stepped.index(False)
    assert not any(stepped[first_off:])


@pytest.mark.parametrize("plant", ["sched_in_warmup", "continue_epoch"])
def test_plan_comparison_catches_a_planted_error(plant):
  c = CASES["fresh_crosses_warmup"]
  planted, _ = literal(*c, **{plant: True})
  assert planted != planned(*c)


def test_plan_steps_match_the_loader_epochs():
  steps = list(tr.plan(7, 20, 4, 0, 5, 5, 5, 1e-4, 28, 0.5))
  by_epoch = {}
  for s in steps:
    by_epoch[(s.phase, s.epoch)] = by_epoch.get((s.phase, s.epoch), 0) + 1
  assert set(by_epoch.values()) == {7}


# ---------------------------------------------------------------------------------------------------------------
# 2. the config file
# ---------------------------------------------------------------------------------------------------------------
KID_RUNNING = """expname = kid-running-test

rootdir = /home/zhengqili/dynibar

folder_path = /home/zhengqili/release

no_reload = False
render_stride = 1
distributed = False
no_load_opt = True
no_load_scheduler = True
n_iters = 400000

## dataset
train_dataset = monocular
train_scenes = kid-running
eval_dataset = monocular
eval_scenes = kid-running

### TRAINING
N_rand = 3072
lrate_feature = 8e-4
lrate_mlp = 4e-4
lrate_decay_factor = 0.5
init_decay_epoch = 400 # modify this s.t. num_imgs * num_epoch ~= 30-40K

### TESTING
chunk_size = 8192

### RENDERING
N_importance = 0
N_samples = 64
inv_uniform = True
white_bkgd = False

### CONSOLE AND TENSORBOARD
i_img = 5000
i_print = 5000
i_weights = 10000

anti_alias_pooling = 0
mask_rgb = 1
input_dir = True
input_xyz = False

training_height = 288

w_cycle = 0.1
cycle_factor = 0.1

w_disp = 1e-1
w_flow = 1e-2
w_distortion = 1e-3
w_reg = 0.05

w_skew_entropy = 5e-4
lr_multipler = 1.0

decay_rate = 10
anneal_cycle = True

erosion_radius = 3
occ_weights_mode = 0

max_range = 42
num_source_views = 7

num_vv = 3
mask_src_view = True
"""


def test_config_file_and_overrides(tmp_path):
  cfg = tmp_path / "train_kid-running.txt"
  cfg.write_text(KID_RUNNING)
  a = train_tool.parse_args(["--config", str(cfg), "--scene_path", "s"])
  assert (a.N_rand, a.lrate_feature, a.lrate_mlp, a.init_decay_epoch, a.chunk_size) == (3072, 8e-4, 4e-4, 400, 8192)
  assert (a.i_img, a.i_print, a.i_weights, a.n_iters, a.N_samples) == (5000, 5000, 10000, 400000, 64)
  assert a.inv_uniform is True and a.input_dir is True and a.anneal_cycle is True and a.mask_src_view is True
  assert a.no_reload is False and a.det is False
  assert (a.anti_alias_pooling, a.mask_rgb, a.erosion_radius, a.max_range, a.num_vv) == (0, 1, 3, 42, 3)
  assert (a.w_disp, a.w_flow, a.w_skew_entropy, a.decay_rate) == (0.1, 0.01, 5e-4, 10.0)
  assert a.rootdir == "/home/zhengqili/dynibar" and a.sample_mode == "uniform" and a.slice_rays == 1024
  assert a.expname == "kid-running-test_mr-42_w-disp-0.100_w-flow-0.010_anneal_cycle-0.1-0.1-w_mode-0"
  b = train_tool.parse_args(["--config", str(cfg), "--scene_path", "s", "--N_rand", "1024", "--rootdir", "/tmp/r",
                             "--no_reload", "--expname", "e"])
  assert b.N_rand == 1024 and b.rootdir == "/tmp/r" and b.no_reload is True and b.lrate_mlp == 4e-4
  assert b.expname.startswith("e_mr-42_")
  d = train_tool.parse_args(["--scene_path", "s"])  # the reference's defaults
  assert (d.N_rand, d.init_decay_epoch, d.lrate_mlp, d.i_print, d.inv_uniform) == (512, 150, 5e-4, 100, False)


@pytest.mark.parametrize("line", ["N_rand = many", "no_such_key = 1", "inv_uniform = maybe", "just a line"])
def test_config_file_rejects_bad_lines(tmp_path, line):
  cfg = tmp_path / "bad.txt"
  cfg.write_text("N_samples = 64\n%s\n" % line)
  with pytest.raises(ValueError):
    train_tool.parse_args(["--config", str(cfg), "--scene_path", "s"])


# ---------------------------------------------------------------------------------------------------------------
# 3.-4. optimiser and checkpoints
# ---------------------------------------------------------------------------------------------------------------
def _args():
  return SimpleNamespace(coarse_feat_dim=32, fine_feat_dim=32, N_samples=16, N_importance=0, num_basis=6,
                         anti_alias_pooling=1, mask_rgb=1, input_dir=True, input_xyz=False, occ_weights_mode=0,
                         lrate_mlp=4e-4, lrate_feature=8e-4, lrate_decay_factor=0.5, init_decay_epoch=3)


def test_optimizer_groups_follow_the_reference():
  a = _args()
  torch.manual_seed(0)
  m = tr.build_model(a, 12, "cpu")
  opt = tr.make_optimizer(m, a)
  want = [(m.net_coarse_st, 2e-4), (m.feature_net_st, 4e-4), (m.net_coarse_dy, 4e-4), (m.feature_net, 8e-4),
          (m.motion_mlp, 4e-4), (m.trajectory_basis, 1e-4)]
  assert len(opt.param_groups) == 6
  for g, (obj, lr) in zip(opt.param_groups, want):
    params = [obj] if torch.is_tensor(obj) else list(obj.parameters())
    assert g["lr"] == pytest.approx(lr, rel=0, abs=1e-18) and len(g["params"]) == len(params)
    assert all(p is q for p, q in zip(g["params"], params))
  assert all(p.requires_grad for g in opt.param_groups for p in g["params"])
  # the reference's initialisation
  assert torch.count_nonzero(m.motion_mlp.coeff_linear.weight) == 0
  assert m.net_coarse_st.s.item() == pytest.approx(0.2) and m.net_coarse_dy.shift == 5.0
  assert torch.equal(m.trajectory_basis.detach(), dmodel.init_dct_basis(6, 12))
  sched = tr.make_scheduler(opt, a, 12)
  assert sched.step_size == 36 and sched.gamma == 0.5


def _stepped(a, seed):
  """A model, optimiser and scheduler after two Adam steps on seeded gradients (every tensor of every group)."""
  torch.manual_seed(seed)
  m = tr.build_model(a, 12, "cpu")
  opt = tr.make_optimizer(m, a)
  sched = tr.make_scheduler(opt, a, 12)
  g = torch.Generator().manual_seed(seed)
  for _ in range(2):
    for grp in opt.param_groups:
      for p in grp["params"]:
        p.grad = torch.randn(p.shape, generator=g) * 1e-2
    opt.step()
    sched.step()
  return m, opt, sched


def test_checkpoint_layout_and_loading(tmp_path):
  a = _args()
  m, opt, sched = _stepped(a, 1)
  loader_rng = np.random.RandomState(11)
  loader_rng.randint(100)
  path = str(tmp_path / "model_latest.pth")
  torch.save(tr.checkpoint(m, opt, sched, 123, tr.rng_state(loader_rng)), path)
  ck = torch.load(path, map_location="cpu", weights_only=False)
  assert sorted(ck) == sorted(tr.CKPT_KEYS + (tr.RNG_KEY,))
  assert set(tr.CKPT_KEYS) == {"optimizer", "scheduler", "net_coarse_st", "net_coarse_dy", "feature_net",
                               "feature_net_st", "motion_mlp", "traj_basis", "global_step"}
  # loadable for rendering
  got, info = dmodel.model_from_checkpoints(a, coarse=path, mono=True)
  assert info["coarse_step"] == 123 and sorted(info["encoders"]) == ["feature_net", "feature_net_st"]
  for k in ("net_coarse_st", "net_coarse_dy", "motion_mlp"):
    for (n1, v1), (n2, v2) in zip(getattr(m, k).state_dict().items(), getattr(got, k).state_dict().items()):
      assert n1 == n2 and torch.equal(v1, v2), (k, n1)
  assert torch.equal(got.trajectory_basis, m.trajectory_basis.detach())
  # the optimizer state into a fresh six-group Adam, and the whole checkpoint into a fresh run
  m2, opt2, sched2 = _stepped(a, 2)
  fresh = torch.optim.Adam([{"params": list(g["params"]), "lr": g["lr"]} for g in opt2.param_groups])
  fresh.load_state_dict(ck["optimizer"])
  assert [g["lr"] for g in fresh.param_groups] == [g["lr"] for g in opt.param_groups]
  rng2 = np.random.RandomState(0)
  sample_ray.rng.randint(5)
  pix = sample_ray.rng.get_state()
  step = tr.load_checkpoint(ck, m2, opt2, sched2)
  tr.set_rng_state(ck[tr.RNG_KEY], rng2)
  assert step == 123 and sched2.last_epoch == sched.last_epoch and sched2.get_last_lr() == sched.get_last_lr()
  assert rng2.randint(1 << 30) == loader_rng.randint(1 << 30)
  assert not np.array_equal(pix[1], sample_ray.rng.get_state()[1]) or pix[2] != sample_ray.rng.get_state()[2]
  for k in tr.NETS:
    for v1, v2 in zip(getattr(m, k).state_dict().values(), getattr(m2, k).state_dict().values()):
      assert torch.equal(v1, v2), k
  assert torch.equal(m2.trajectory_basis, m.trajectory_basis) and m2.trajectory_basis is opt2.param_groups[5]["params"][0]
  for p1, p2 in zip([p for g in opt.param_groups for p in g["params"]], [p for g in opt2.param_groups for p in g["params"]]):
    s1, s2 = opt.state[p1], opt2.state[p2]
    assert torch.equal(s1["step"], s2["step"]) and torch.equal(s1["exp_avg"], s2["exp_avg"])
    assert torch.equal(s1["exp_avg_sq"], s2["exp_avg_sq"])


def test_resume_search_follows_load_from_ckpt(tmp_path):
  out = tmp_path / "out"
  out.mkdir()
  a = SimpleNamespace(pretrain_path="", ckpt_path="", no_reload=False)
  assert tr.find_checkpoint(a, str(out)) is None
  for name in ("model_no-vv.pth", "a_latest.pth", "model_latest.pth"):
    (out / name).write_bytes(b"")
  assert tr.find_checkpoint(a, str(out)) == str(out / "model_latest.pth")
  other = tmp_path / "given.pth"
  other.write_bytes(b"")
  a.ckpt_path = str(other)
  assert tr.find_checkpoint(a, str(out)) == str(other)
  a.no_reload = True
  assert tr.find_checkpoint(a, str(out)) is None
