"""train.py's monocular training loop (train.py:47-573) and DynibarMono's model, optimiser, scheduler and checkpoints
(ibrnet/model.py:291-501) as a library.

  trainer = Trainer(args, scene, device)       # nets from scratch, or resumed as load_from_ckpt does
  trainer.run()                                # the warm-up and the main phase, as `plan` lays them out

`plan` restates the loop's control flow on the host alone: which phase and epoch each step is in, the global step it
logs under, whether the scheduler steps and which actions (print, render the training view, save) follow.  The loop
runs that plan and nothing else decides its control flow.  A step is one `train_step.mono_step_backward` (the batch in
ray slices; `bootstrap=True` in the warm-up) between `zero_grad` and `optimizer.step()`; its loss terms stay on the
device and are read back only on print steps.

Checkpoints have DynibarMono.save_model's keys plus RNG_KEY, the state of the loop's draws (the scene's RandomState, the
pixel RandomState `sample_ray.rng` and the CUDA generator that draws the samples' jitter), so that a resumed run draws
what an uninterrupted one would.  The reference never reads that key, and `model.model_from_checkpoints(mono=True)`
ignores it.  One deliberate difference on resume: the reference's load_model rebinds `trajectory_basis` to the loaded
tensor, which is not the one its optimiser holds, so a resumed reference run stops training the basis; here the loaded
values are copied into the optimised tensor.
"""

import collections
import os
import time
from types import SimpleNamespace

import numpy as np
import torch

from dynibar_b200 import mlp_network as nets
from dynibar_b200 import model as dmodel
from dynibar_b200 import sample_ray
from dynibar_b200 import train_step as ts
from dynibar_b200.feature_network import ResNet

WARMUP, MAIN = "warmup", "main"
PRINT, RENDER, SAVE_LATEST, SAVE_NO_VV = "print", "render", "save_latest", "save_no_vv"
LR_FLOOR = 5e-7            # train.py:469: the scheduler steps only while the first group's lr is above this
MAX_EPOCH = 10 ** 5        # train.py:227
NETS = ("net_coarse_st", "net_coarse_dy", "feature_net", "feature_net_st", "motion_mlp")
CKPT_KEYS = ("optimizer", "scheduler") + NETS + ("traj_basis", "global_step")
RNG_KEY = "loop_rng_state"
# the optimiser's parameter groups in the reference's order (the checkpoint's optimizer state is indexed by it) and
# each group's learning rate as (option, factor) (ibrnet/model.py:341-351)
GROUPS = (("net_coarse_st", "lrate_mlp", 0.5), ("feature_net_st", "lrate_feature", 0.5),
          ("net_coarse_dy", "lrate_mlp", 1.0), ("feature_net", "lrate_feature", 1.0),
          ("motion_mlp", "lrate_mlp", 1.0), ("trajectory_basis", "lrate_mlp", 0.25))

Step = collections.namedtuple("Step", "phase epoch global_step sched_step lr actions")
Step.__doc__ = """One step of the loop.  global_step: the value the step logs and saves under (the warm-up adds 1
before, the main phase after).  sched_step: whether scheduler.step() follows optimizer.step().  lr: the first group's
learning rate after the step (what train.py:472 logs).  actions: a tuple of PRINT, RENDER, SAVE_LATEST, SAVE_NO_VV."""


def plan(num_frames, n_iters, init_decay_epoch, start_step, i_print, i_img, i_weights, lr, step_size, gamma,
         sched_epoch=0):
  """The steps of train.py:111-573 from `start_step`, in order (a generator).

  lr, sched_epoch: the scheduler's get_last_lr()[0] and last_epoch when the loop starts; step_size, gamma: StepLR's.
  Restated with the reference's quirks: the warm-up runs epochs start_epoch .. init_decay_epoch // 2 - 1 with
  start_epoch = start_step // num_frames, never steps the scheduler, and only renders; the main phase starts again
  from start_epoch (the criterion's epoch restarts), and stops when global_step > start_step + n_iters + 1 at the
  start of an epoch.  model_no-vv.pth is saved at the first step of epoch init_decay_epoch * 5 - 1."""
  gs = start_step
  start_epoch = gs // num_frames
  for epoch in range(start_epoch, init_decay_epoch // 2):
    for _ in range(num_frames):
      gs += 1
      yield Step(WARMUP, epoch, gs, False, lr, (RENDER,) if gs % i_img == 0 else ())
  no_vv_saved = False
  for epoch in range(start_epoch, MAX_EPOCH):
    if gs > start_step + n_iters + 1:
      return
    for _ in range(num_frames):
      sched = lr > LR_FLOOR
      if sched:  # StepLR.step: last_epoch += 1, the lr times gamma at every multiple of step_size
        sched_epoch += 1
        if sched_epoch % step_size == 0:
          lr = lr * gamma
      actions = []
      if epoch + 1 == init_decay_epoch * 5 and not no_vv_saved:
        actions.append(SAVE_NO_VV)
        no_vv_saved = True
      if gs % i_print == 0:
        actions.append(PRINT)
      if gs % i_weights == 0:
        actions.append(SAVE_LATEST)
      if gs % i_img == 0:
        actions.append(RENDER)
      yield Step(MAIN, epoch, gs, sched, lr, tuple(actions))
      gs += 1


# ---- model, optimiser, scheduler, checkpoints (ibrnet/model.py:294-364, :424-501) -----------------------------------

def build_model(args, num_frames, device):
  """DynibarMono's nets from scratch, every tensor requiring grad: torch's default nn.Linear / Conv2d init (the
  reference's weights_init is never applied), coeff_linear zeroed, s = 0.2 with anti_alias_pooling, the DCT basis."""
  m = SimpleNamespace()
  m.net_coarse_st = nets.DynibarStatic(args, args.coarse_feat_dim, args.N_samples).to(device)
  m.net_coarse_dy = nets.DynibarDynamic(args, args.coarse_feat_dim, args.N_samples, shift=5.0).to(device)
  m.feature_net = ResNet(coarse_out_ch=args.coarse_feat_dim, fine_out_ch=args.fine_feat_dim,
                         coarse_only=False).to(device)
  m.feature_net_st = ResNet(coarse_out_ch=args.coarse_feat_dim, fine_out_ch=args.fine_feat_dim,
                            coarse_only=False).to(device)
  m.motion_mlp = nets.MotionMLP(num_basis=args.num_basis).float().to(device)
  m.trajectory_basis = dmodel.init_dct_basis(args.num_basis, num_frames).to(device).requires_grad_(True)
  for k in NETS:
    getattr(m, k).requires_grad_(True)
  return m


def make_optimizer(model, args):
  """torch.optim.Adam over the six groups of GROUPS."""
  groups = []
  for name, opt, factor in GROUPS:
    obj = getattr(model, name)
    params = [obj] if torch.is_tensor(obj) else list(obj.parameters())
    groups.append({"params": params, "lr": getattr(args, opt) * factor})
  return torch.optim.Adam(groups)


def make_scheduler(optimizer, args, num_frames):
  """StepLR(step_size = num_frames * init_decay_epoch, gamma = lrate_decay_factor) (train.py:92, model.py:360)."""
  return torch.optim.lr_scheduler.StepLR(optimizer, step_size=num_frames * args.init_decay_epoch,
                                         gamma=args.lrate_decay_factor)


def rng_state(loader_rng, device=None):
  """The loop's draws: the scene's RandomState, sample_ray.rng (pixels) and, on a CUDA device, its generator."""
  st = {"loader": loader_rng.get_state(), "pixels": sample_ray.rng.get_state()}
  if device is not None and torch.device(device).type == "cuda":
    st["cuda"] = torch.cuda.get_rng_state(device)
  return st


def set_rng_state(st, loader_rng, device=None):
  loader_rng.set_state(st["loader"])
  sample_ray.rng.set_state(st["pixels"])
  if "cuda" in st and device is not None and torch.device(device).type == "cuda":
    torch.cuda.set_rng_state(st["cuda"].cpu(), device)


def checkpoint(model, optimizer, scheduler, global_step, rng=None):
  """DynibarMono.save_model's dict (ibrnet/model.py:424-441), plus RNG_KEY when `rng` (rng_state's dict) is given."""
  ck = {"optimizer": optimizer.state_dict(), "scheduler": scheduler.state_dict()}
  for k in NETS:
    ck[k] = getattr(model, k).state_dict()
  ck["traj_basis"] = model.trajectory_basis.detach()
  ck["global_step"] = int(global_step)
  if rng is not None:
    ck[RNG_KEY] = rng
  return ck


def load_checkpoint(ck, model, optimizer, scheduler):
  """DynibarMono.load_model with load_opt and load_scheduler (ibrnet/model.py:443-466) -> global_step.  The basis is
  copied into the optimised tensor (see the module docstring)."""
  optimizer.load_state_dict(ck["optimizer"])
  scheduler.load_state_dict(ck["scheduler"])
  for k in NETS:
    getattr(model, k).load_state_dict(dmodel._strip(ck[k]))
  with torch.no_grad():
    model.trajectory_basis.copy_(ck["traj_basis"])
  return int(ck["global_step"])


def find_checkpoint(args, out_folder):
  """The file load_from_ckpt resumes from (ibrnet/model.py:370-378, :468-500), or None: `ckpt_path` when it is a
  file, else the last by name of the files ending in latest.pth in `pretrain_path` (when set) or `out_folder`; None
  with no_reload."""
  folder = args.pretrain_path or out_folder
  ckpts = []
  if folder and os.path.isdir(folder):
    ckpts = [os.path.join(folder, f) for f in sorted(os.listdir(folder)) if f.endswith("latest.pth")]
  if args.ckpt_path and os.path.isfile(args.ckpt_path):
    ckpts = [args.ckpt_path]
  if ckpts and not args.no_reload:
    return ckpts[-1]
  return None


# ---- the loop ------------------------------------------------------------------------------------------------------

def _grey(x):
  """[H, W] -> [H, W] in [0, 1], min-max normalised."""
  lo, hi = x.min(), x.max()
  return (x - lo) / (hi - lo) if hi > lo else torch.zeros_like(x)


class Trainer(object):
  """One monocular training run on one device.

  args: the reference's config names the loop reads (tools/train.py lists them); `slice_rays` (default 1024) is the
  ray slice of mono_step_backward.  scene: a MonocularScene.  out_folder: where checkpoints, PNGs and the resume
  search go (None: nothing is resumed; saves need an explicit path).  seed: the scene's RandomState (the reference's
  loader workers seed np.random from the OS).  log: a callable taking one line of text."""

  def __init__(self, args, scene, device, out_folder=None, seed=0, log=print):
    self.args, self.scene, self.device = args, scene, torch.device(device)
    self.out_folder, self.log = out_folder, log
    self.num_frames = scene.num_frames
    self.slice_rays = int(getattr(args, "slice_rays", 1024))
    self.model = build_model(args, self.num_frames, self.device)
    self.optimizer = make_optimizer(self.model, args)
    self.scheduler = make_scheduler(self.optimizer, args, self.num_frames)
    self.rng = np.random.RandomState(seed)
    from dynibar_b200.projection import Projector
    self.projector = Projector(self.device)
    self.start_step = 0
    path = find_checkpoint(args, out_folder) if out_folder is not None or args.ckpt_path else None
    if path is not None:
      self.start_step = self.load(path)
      log("Reloading from %s, starting at step=%d" % (path, self.start_step))
    else:
      log("No ckpts found, training from scratch...")
    self.global_step = self.start_step
    self.writer = None
    self.step_times = []  # host time from one step's start to the next's
    self.windows = []     # (global_step, steps, median step time) per print
    self._mark = 0
    self._steps, self._epoch, self._draws, self._t_prev = None, None, None, None

  # -- checkpoints --
  def save(self, path, global_step):
    torch.save(checkpoint(self.model, self.optimizer, self.scheduler, global_step,
                          rng_state(self.rng, self.device)), path)

  def load(self, path):
    ck = torch.load(path, map_location=self.device, weights_only=False)
    step = load_checkpoint(ck, self.model, self.optimizer, self.scheduler)
    if RNG_KEY in ck:
      set_rng_state(ck[RNG_KEY], self.rng, self.device)
    return step

  # -- one step --
  def plan(self):
    a = self.args
    return plan(self.num_frames, a.n_iters, a.init_decay_epoch, self.start_step, a.i_print, a.i_img, a.i_weights,
                self.scheduler.get_last_lr()[0], self.scheduler.step_size, self.scheduler.gamma,
                self.scheduler.last_epoch)

  def batch(self, train_data):
    """frame ids, time embeddings and time offsets of a batch (train.py:236-254; the ids are read back, as there)."""
    i, an = int(train_data["id"]), int(train_data["anchor_id"])
    offs = ([int(j) - i for j in train_data["nearest_pose_ids"][0]],
            [int(j) - an for j in train_data["anchor_nearest_pose_ids"][0]])
    return (i, an), (train_data["ref_time"], train_data["anchor_time"]), offs

  def featmaps(self, rb, bootstrap):
    """The encoders' coarse maps of the three stacks (train.py:150-167).  The warm-up renders with is_train=False,
    which never reads the anchor stack's maps, so they are not computed there."""
    enc = lambda net, k: net(rb[k][0].permute(0, 3, 1, 2).contiguous())[0]
    m = self.model
    return (enc(m.feature_net, "src_rgbs"), None if bootstrap else enc(m.feature_net, "anchor_src_rgbs"),
            enc(m.feature_net_st, "static_src_rgbs"))

  def step(self, train_data, rb, epoch, bootstrap, sched_step):
    """zero_grad, mono_step_backward, optimizer.step() and, when `sched_step`, scheduler.step() -> (loss, terms) on the
    device."""
    a = self.args
    frame, t, offs = self.batch(train_data)
    fm = self.featmaps(rb, bootstrap)
    self.optimizer.zero_grad()
    loss, terms = ts.mono_step_backward(frame, t, offs, rb, self.model, fm, self.projector, a.N_samples, a, epoch,
                                        slice_rays=self.slice_rays, bootstrap=bootstrap, inv_uniform=a.inv_uniform,
                                        det=a.det, num_vv=a.num_vv)
    self.optimizer.step()
    if sched_step:
      self.scheduler.step()
    return loss, terms

  def run(self, max_steps=None):
    """Runs the plan, or its next `max_steps` steps (a later call continues where this one stopped) -> the number of
    steps run."""
    a = self.args
    if self._steps is None:
      self._steps = self.plan()
    n = 0
    while max_steps is None or n < max_steps:
      st = next(self._steps, None)
      if st is None:
        break
      if (st.phase, st.epoch) != self._epoch:  # a new epoch of the loader: train_dataset.set_epoch, then one pass
        self._epoch = (st.phase, st.epoch)
        self.scene.set_epoch(st.epoch)
        self._draws = self.scene.loader(self.rng, a.N_rand, a.sample_mode)
        self.log(("================ Static Boostrap %d" if st.phase == WARMUP else "====================================== %d")
                 % st.epoch)
      t0 = time.perf_counter()
      if self._t_prev is not None:
        # the step reads cameras and times back before its first kernels, so the host cannot run a step ahead
        self.step_times.append(t0 - self._t_prev)
      self._t_prev = t0
      train_data, rb = next(self._draws)
      _, terms = self.step(train_data, rb, st.epoch, st.phase == WARMUP, st.sched_step)
      self.global_step = st.global_step if st.phase == WARMUP else st.global_step + 1
      n += 1
      if SAVE_NO_VV in st.actions:
        path = os.path.join(self.out_folder, "model_no-vv.pth")
        if not os.path.exists(path):
          self.save(path, st.global_step)
      if PRINT in st.actions:
        self._print(st, terms)
      if SAVE_LATEST in st.actions:
        self.log("Saving checkpoints at %d to %s..." % (st.global_step, self.out_folder))
        self.save(os.path.join(self.out_folder, "model_latest.pth"), st.global_step)
      if RENDER in st.actions:
        self.render_view(train_data, st.global_step)
    return n

  # -- logging --
  def _writer(self):
    if self.writer is None:
      try:
        from torch.utils.tensorboard import SummaryWriter
      except ImportError:
        self.writer = False
      else:
        self.writer = SummaryWriter(os.path.join(self.args.rootdir, "logs", self.args.expname))
    return self.writer

  def _print(self, st, terms):
    names = list(terms)
    vals = torch.stack([terms[k] for k in names]).tolist()  # the step's one read-back
    scalars = dict(zip(names, vals), lr=self.scheduler.get_last_lr()[0])
    window = self.step_times[self._mark:]
    self._mark = len(self.step_times)
    med = float(np.median(window)) if window else float("nan")
    self.windows.append((st.global_step, len(window), med))
    self.log("%s Epoch: %d  step: %d %s  median step time %.5f seconds over %d steps"
             % (self.args.expname, st.epoch, st.global_step,
                " ".join("%s: %.6f" % kv for kv in scalars.items()), med, len(window)))
    w = self._writer()
    if w:
      for k, v in scalars.items():
        w.add_scalar(k, v, st.global_step)

  def render_view(self, train_data, global_step):
    """log_view_to_tb (train.py:576-762) without flows: the training view rendered with is_train=True, det=True under
    no_grad, written as PNGs under <out_folder>/train_views/<global_step>/ -> that folder."""
    import cv2
    from dynibar_b200.render_image import render_single_image_mono
    a, m = self.args, self.model
    frame, t, offs = self.batch(train_data)
    with torch.no_grad():
      rb = self.scene.get_all(train_data)
      fm = (m.feature_net(rb["src_rgbs"][0].permute(0, 3, 1, 2).contiguous())[0],
            m.feature_net(rb["anchor_src_rgbs"][0].permute(0, 3, 1, 2).contiguous())[0],
            m.feature_net_st(rb["static_src_rgbs"][0].permute(0, 3, 1, 2).contiguous())[0])
      ret = render_single_image_mono(frame, t, offs, SimpleNamespace(H=self.scene.H, W=self.scene.W), rb, m,
                                     self.projector, a.chunk_size, a.N_samples, a, inv_uniform=a.inv_uniform,
                                     det=True, featmaps=fm, is_train=True, num_vv=a.num_vv)
    ref, anc, st = ret["outputs_coarse_ref"], ret["outputs_coarse_anchor"], ret["outputs_coarse_st"]
    images = {"render_rgb_coarse_ref": ref["rgb"], "render_rgb_coarse_anchor": anc["rgb"],
              "render_rgb_static": ref["rgb_static"], "render_rgb_dynamic": ref["rgb_dy"], "st_rgb_pred": st["rgb"],
              "gt_rgb_coarse": train_data["rgb"][0].cpu(), "render_depth_coarse": _grey(ref["depth"]),
              "occ_weight_map": _grey(anc["occ_weight_map"])}
    d = os.path.join(self.out_folder, "train_views", "%06d" % global_step)
    os.makedirs(d, exist_ok=True)
    w = self._writer()
    for name, x in images.items():
      x = x.float().clamp(0.0, 1.0)
      u8 = (x * 255.0 + 0.5).to(torch.uint8).numpy()
      cv2.imwrite(os.path.join(d, name + ".png"), u8[..., ::-1] if u8.ndim == 3 else u8)
      if w:
        w.add_image("train/" + name, x.permute(2, 0, 1) if x.dim() == 3 else x[None], global_step)
    return d
