"""Generate golden fixtures by running the UNMODIFIED reference on CPU.

Run in the build container (where /root/reference exists):

    python tests/golden/make_golden.py

Writes tests/golden/*.pt.  The fixtures hold only reference OUTPUTS (and the
stage-boundary tensors) -- inputs and weights are regenerated from the same
seeds by `dynibar_b200.synthetic` / `tests/scenes.py`, and an input checksum in
each fixture guards against RNG drift.  Nothing here is imported by the
product.
"""

import os
import sys
import types
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REF = os.environ.get("DYNIBAR_REFERENCE", "/root/reference")  # as in oracle/build_ref.py
# the gather outputs rgb_feat_* [R,S,V,35] dominate a fixture: they are stored for every STAGE_RAY_STEP-th ray
# only (whole rays: the networks couple the samples of a ray), which keeps each fixture under 1 MB
STAGE_RAY_STEP = 3

warnings.filterwarnings("ignore")


def import_reference():
  """Import the reference's hot-path modules unmodified (SURVEY App. C)."""
  if REF not in sys.path:
    sys.path.insert(0, REF)
  if "kornia" not in sys.modules:  # only create_meshgrid is used (sample_ray.py:6,83)
    k = types.ModuleType("kornia")

    def create_meshgrid(H, W, normalized_coordinates=False):
      ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32),
                              torch.arange(W, dtype=torch.float32), indexing="ij")
      return torch.stack([xs, ys], -1)[None]

    k.create_meshgrid = create_meshgrid
    sys.modules["kornia"] = k
  from ibrnet import mlp_network, projection, render_ray, sample_ray  # noqa
  return types.SimpleNamespace(mlp=mlp_network, proj=projection, rr=render_ray,
                               sr=sample_ray)


def reference_model(ref, model, args, mono):
  """Reference nn.Modules carrying the weights of our mirror containers
  (also proves the state_dict names/shapes line up: strict load)."""
  out = types.SimpleNamespace()

  def conv(m):
    name = type(m).__name__
    if name == "DynibarDynamic":
      r = ref.mlp.DynibarDynamic(args, m.in_feat_ch, m.n_samples, shift=m.shift)
    elif name == "DynibarStatic":
      r = ref.mlp.DynibarStatic(args, m.in_feat_ch, m.n_samples)
    else:
      r = ref.mlp.MotionMLP(num_basis=m.num_basis)
    r.load_state_dict(m.state_dict(), strict=True)
    return r.eval()

  for k, v in vars(model).items():
    setattr(out, k, conv(v) if isinstance(v, torch.nn.Module) else v)
  return out


def checksum(batch, feats):
  acc = 0.0
  for k in sorted(batch):
    if torch.is_tensor(batch[k]):
      acc += float(batch[k].double().abs().sum())
  for f in feats:
    for x in f:
      if x is not None:
        acc += float(x.double().abs().sum())
  return acc


def stage_tensors(ref, batch, feat, model_ref, args, frame, t, offs, S, num_vv,
                  inv_uniform):
  """Stage-boundary tensors of ONE coarse pass, produced by calling the
  reference's own component functions (render_ray.py:660-782 sequence)."""
  rr = ref.rr
  P = ref.proj.Projector("cpu")
  pts, z, s = rr.sample_along_camera_ray(batch["ray_o"], batch["ray_d"],
                                         batch["depth_range"], S,
                                         inv_uniform=inv_uniform, det=True)
  R = pts.shape[0]
  te = t[0][None, None, :].repeat(R, S, 1)
  xyzt = torch.cat([pts, te], -1).float()
  coeff = model_ref.motion_mlp(xyzt)
  n_last = int(round(S * 0.1))
  coeff[:, -n_last:, :] *= 0.0
  nb = model_ref.trajectory_basis.shape[1]
  traj = {}
  for o in range(-3, 4):
    traj[o] = rr.compute_traj_pts(coeff[..., :nb], coeff[..., nb:2 * nb],
                                  coeff[..., 2 * nb:],
                                  model_ref.trajectory_basis[None, None, frame[0] + o, :])
  seq = [pts + (traj[o] - traj[0]) for o in offs[0]] + [pts] * num_vv
  seq = torch.stack(seq, 0)
  V_st = batch["static_src_rgbs"].shape[1]
  f_dy, rd_dy, m_dy = P.compute_with_motions(pts, seq, batch["camera"],
                                             batch["src_rgbs"],
                                             batch["src_cameras"], feat[0])
  f_st, rd_st, m_st = P.compute_with_motions(pts, pts[None].repeat(V_st, 1, 1, 1),
                                             batch["camera"],
                                             batch["static_src_rgbs"],
                                             batch["static_src_cameras"], feat[2])
  ray_dir = torch.nn.functional.normalize(batch["ray_d"], dim=-1)
  raw_dy = model_ref.net_coarse_dy(pts, f_dy.clone(), ray_dir, rd_dy, None, m_dy, te)
  ref_pl = rr.compute_ref_plucker_coordinate(batch["ray_o"], batch["ray_d"])
  src_pl = rr.compute_src_plucker_coordinate(pts, batch["static_src_cameras"])
  raw_st = model_ref.net_coarse_st(pts, ref_pl, src_pl, f_st.clone(), ray_dir,
                                   rd_st, m_st)
  return dict(pts=pts, z=z, s=s, coeff=coeff, seq=seq, rgb_feat_dy=f_dy,
              ray_diff_dy=rd_dy, mask_dy=m_dy, rgb_feat_st=f_st,
              ray_diff_st=rd_st, mask_st=m_st, raw_dy=raw_dy, raw_st=raw_st,
              ref_plucker=ref_pl, src_plucker=src_pl)


def sample_stage_rays(st):
  """keep rgb_feat_dy / rgb_feat_st for the rays rgb_feat_rays only"""
  rays = torch.arange(0, st["rgb_feat_dy"].shape[0], STAGE_RAY_STEP)
  st["rgb_feat_rays"] = rays
  for k in ("rgb_feat_dy", "rgb_feat_st"):
    st[k] = st[k][rays].clone()
  return st


def clean(d):
  if d is None:
    return None
  return {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in d.items()}


def main():
  import scenes
  ref = import_reference()
  torch.set_grad_enabled(False)
  for name, cfg in scenes.GOLDEN_CONFIGS.items():
    batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
    mref = reference_model(ref, model, args, cfg["mono"])
    P = ref.proj.Projector("cpu")
    fx = {"cfg": cfg, "checksum": checksum(batch, [feat_c, feat_f])}
    if cfg["mono"]:
      train = cfg.get("anchor_offset") is not None
      ret = ref.rr.render_rays_mono(frame, t, offs, batch, mref, feat_c, P,
                                    cfg["N_samples"], args,
                                    inv_uniform=cfg["inv_uniform"], det=True,
                                    is_train=train, num_vv=cfg["num_vv"])
      keys = ("outputs_coarse_ref", "outputs_coarse_ref_dy", "outputs_coarse_st")
      if train:
        keys += ("outputs_coarse_anchor", "outputs_coarse_anchor_dy")
      for k in keys:
        fx[k] = clean(ret[k])
    else:
      ret = ref.rr.render_rays_mv(frame, t, offs, batch, mref, P, feat_c, feat_f,
                                  cfg["N_samples"], args,
                                  inv_uniform=cfg["inv_uniform"],
                                  N_importance=cfg["N_importance"], det=True,
                                  is_train=False)
      for k in ("outputs_coarse_ref", "outputs_fine_ref", "outputs_fine_ref_dy"):
        fx[k] = clean(ret[k])
      # non-deterministic sampling: same torch RNG stream as the reference
      torch.manual_seed(cfg["seed"] + 1000)
      ret = ref.rr.render_rays_mv(frame, t, offs, batch, mref, P, feat_c, feat_f,
                                  cfg["N_samples"], args,
                                  inv_uniform=cfg["inv_uniform"],
                                  N_importance=cfg["N_importance"], det=False,
                                  is_train=False)
      fx["rand_outputs_fine_ref"] = clean(ret["outputs_fine_ref"])
    fx["stages"] = sample_stage_rays(clean(stage_tensors(ref, batch, feat_c, mref, args, frame, t,
                                                         offs, cfg["N_samples"], cfg["num_vv"],
                                                         cfg["inv_uniform"])))
    path = os.path.join(HERE, name + ".pt")
    torch.save(fx, path)
    print(name, "->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
  main()
