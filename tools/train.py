#!/usr/bin/env python
"""train.py: train a monocular scene on one GPU (dynibar_b200.trainer), from the device-resident scene.

  python tools/train.py --config configs/train_kid-running.txt --scene_path <folder_path>/<scene>/dense \\
      [--rootdir .] [--expname exp] [--n_iters 400000] [--slice_rays 1024] [any option below]

The options are the keys of the reference's config.py that the loop reads, with its defaults.  `--config FILE` reads
the reference's `key = value` files (`#` comments, booleans as True / False / 0 / 1); options given on the command line
override the file.  The file's other keys of config.py (folder_path, train_scenes, distributed, no_load_opt, ...) are
accepted and not used; the checkpoint's optimizer and scheduler states are always loaded on resume, as DynibarMono does.
The experiment name gets train.py's suffix; out/<expname> under --rootdir holds args.txt, config.txt, model_latest.pth,
model_no-vv.pth and the rendered training views (train_views/<step>/*.png); logs/<expname> holds tensorboard scalars
and images when tensorboard is installed.  At every print step the median step time of the window since the last print
is logged; at the end one JSON line gives every window's median and the card's name and power limit.
"""

import argparse
import json
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

# keys of the reference's config.py the loop does not read: accepted in a config file, ignored
UNUSED_KEYS = ("folder_path", "coarse_dir", "distributed", "local_rank", "workers", "mask_static", "lr_multipler",
               "eval_dataset", "eval_scenes", "render_idx", "train_dataset", "train_scenes", "N_importance",
               "no_load_opt", "no_load_scheduler", "lrate_decay_steps", "w_entropy", "white_bkgd", "render_stride",
               "input_xyz")


def parser():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  add = ap.add_argument
  flag = lambda name, **kw: add(name, action="store_true", **kw)
  add("--config", help="a config file of the reference's key = value form")
  add("--scene_path", required=True, help="the reference's <folder_path>/<scene>/dense")
  add("--rootdir", default=".")
  add("--expname", default="exp")
  add("--device", default="cuda:0")
  add("--seed", type=int, default=0, help="seed of the scene's RandomState (the reference's workers draw one)")
  add("--slice_rays", type=int, default=1024, help="rays per forward / backward slice of a step")
  # data
  add("--training_height", type=int, default=288)
  flag("--mask_src_view")
  add("--N_rand", type=int, default=32 * 16)
  add("--sample_mode", default="uniform")
  add("--num_vv", type=int, default=3)
  add("--erosion_radius", type=int, default=1)
  add("--max_range", type=int, default=35)
  add("--num_source_views", type=int, default=7)
  # loss
  add("--cycle_factor", type=float, default=0.1)
  flag("--anneal_cycle")
  add("--decay_rate", type=float, default=10.0)
  add("--init_decay_epoch", type=int, default=150)
  add("--w_cycle", type=float, default=0.1)
  add("--w_distortion", type=float, default=1e-3)
  add("--w_disp", type=float, default=5e-2)
  add("--w_flow", type=float, default=5e-3)
  add("--w_skew_entropy", type=float, default=1e-3)
  add("--w_reg", type=float, default=0.05)
  add("--occ_weights_mode", type=int, default=0)
  # model and rendering
  add("--chunk_size", type=int, default=1024 * 4)
  add("--coarse_feat_dim", type=int, default=32)
  add("--fine_feat_dim", type=int, default=32)
  add("--num_basis", type=int, default=6)
  add("--anti_alias_pooling", type=int, default=1)
  add("--mask_rgb", type=int, default=1)
  add("--N_samples", type=int, default=64)
  flag("--inv_uniform")
  flag("--input_dir")
  flag("--det")
  # checkpoints and schedule
  flag("--no_reload")
  add("--ckpt_path", default="")
  add("--pretrain_path", default="")
  add("--n_iters", type=int, default=300000)
  add("--lrate_feature", type=float, default=1e-3)
  add("--lrate_mlp", type=float, default=5e-4)
  add("--lrate_decay_factor", type=float, default=0.5)
  # logging
  add("--i_print", type=int, default=100)
  add("--i_img", type=int, default=1000)
  add("--i_weights", type=int, default=10000)
  return ap


def read_config(path, ap):
  """The reference's key = value file -> {dest: value} for `ap`'s options (configargparse's default format)."""
  actions = {a.dest: a for a in ap._actions}
  out = {}
  with open(path) as f:
    for n, line in enumerate(f, 1):
      line = line.strip()
      if not line or line.startswith("#"):
        continue
      if "=" not in line:
        raise ValueError("%s:%d: not a key = value line: %r" % (path, n, line))
      key, value = (s.strip() for s in line.split("=", 1))
      value = value.split(" #")[0].split("\t#")[0].strip()
      if key in UNUSED_KEYS:
        continue
      a = actions.get(key)
      if a is None or key in ("config", "help"):
        raise ValueError("%s:%d: unknown option %r" % (path, n, key))
      if isinstance(a, argparse._StoreTrueAction):
        if value.lower() not in ("true", "false", "1", "0"):
          raise ValueError("%s:%d: %s takes True / False / 1 / 0, got %r" % (path, n, key, value))
        out[key] = value.lower() in ("true", "1")
      else:
        out[key] = (a.type or str)(value)
  return out


def parse_args(argv=None):
  ap = parser()
  pre = argparse.ArgumentParser(add_help=False)
  pre.add_argument("--config")
  known, _ = pre.parse_known_args(argv)
  if known.config:
    ap.set_defaults(**read_config(known.config, ap))
  args = ap.parse_args(argv)
  args.input_dir = bool(args.input_dir)
  args.expname = (args.expname + "_mr-%d" % args.max_range + "_w-disp-%.3f" % args.w_disp
                  + "_w-flow-%.3f" % args.w_flow + "_anneal_cycle-%.1f-%.1f" % (args.w_cycle, args.cycle_factor)
                  + "-w_mode-%d" % args.occ_weights_mode)  # train.py:50-56
  return args


def card(device):
  import torch
  info = {"name": torch.cuda.get_device_name(device)}
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                          "--id=%d" % torch.device(device).index], capture_output=True, text=True, timeout=30)
    power, sm_max = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
    info.update(power_limit=power, sm_max_clock=sm_max)
  except Exception as e:  # nvidia-smi missing: say so instead of guessing
    info.update(power_limit=None, sm_max_clock=None, query_error=repr(e))
  return info


def main(argv=None):
  args = parse_args(argv)
  import torch
  from dynibar_b200 import mono_scene, trainer
  dev = torch.device(args.device)
  if dev.index is None:
    dev = torch.device("cuda", 0)
  torch.cuda.set_device(dev)
  out_folder = os.path.join(args.rootdir, "out", args.expname)
  print("outputs will be saved to {}".format(out_folder))
  os.makedirs(out_folder, exist_ok=True)
  with open(os.path.join(out_folder, "args.txt"), "w") as f:
    for k in sorted(vars(args)):
      f.write("{} = {}\n".format(k, getattr(args, k)))
  if args.config is not None and not os.path.isfile(os.path.join(out_folder, "config.txt")):
    shutil.copy(args.config, os.path.join(out_folder, "config.txt"))
  scene = mono_scene.MonocularScene(args.scene_path, args, dev)
  args.num_frames = scene.num_frames
  args.lrate_decay_steps = args.num_frames * args.init_decay_epoch
  tr = trainer.Trainer(args, scene, dev, out_folder=out_folder, seed=args.seed)
  steps = tr.run()
  torch.cuda.synchronize(dev)
  print(json.dumps({"what": "tools/train.py: %d steps from global step %d, N_rand %d in slices of %d, %d samples"
                            % (steps, tr.start_step, args.N_rand, args.slice_rays, args.N_samples),
                    "print_windows": [{"global_step": g, "steps": n, "median_step_ms": round(m * 1e3, 2)}
                                      for g, n, m in tr.windows],
                    "card": card(dev)}))
  return tr


if __name__ == "__main__":
  main()
