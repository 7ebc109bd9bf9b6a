"""tests/golden/live_reference.pt: outputs of the unmodified reference for the comparisons that need more than
make_golden.py's scenes (run where the reference is, as make_golden.py):

    python tests/golden/make_golden_live.py

mv77: render_rays_mv on a further seeded scene (test_oracle_golden.py); sampler91: RaySamplerSingleImage.get_all
(test_sample_ray_cpu.py); ckpt: key / shape order of the reference modules' state_dicts (test_checkpoint_cpu.py);
encoder: ResNet outputs at three image sizes, a seeded sample of ENCODER_SAMPLES positions (test_encoder_gpu.py).
Inputs are regenerated from seeds by the tests.
"""

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))

ENCODER_SHAPES = [(2, 288, 512), (3, 37, 53), (1, 135, 240)]
ENCODER_SAMPLES = 16384
MV77 = dict(seed=77, rays=16, V_dy=7, V_st=4)
SAMPLER91 = dict(H=17, W=23, rays=None, seed=91)


def encoder_input(N, H, W):
  return torch.rand(N, 3, H, W, generator=torch.Generator().manual_seed(N * 1000 + H + 1))


def encoder_sample(numel, N, H):
  """indices of the stored positions of a flattened encoder output"""
  n = min(numel, ENCODER_SAMPLES)
  return torch.randperm(numel, generator=torch.Generator().manual_seed(N * 1000 + H + 2))[:n]


def checkpoint_args():
  """the arguments tests/test_checkpoint_cpu.py builds its containers with"""
  from dynibar_b200 import synthetic
  a = synthetic.make_args(1, 0)
  a.N_samples, a.N_importance, a.coarse_feat_dim, a.fine_feat_dim = 16, 16, 32, 32
  return a


def main():
  for p in (HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))):
    sys.path.insert(0, p)
  import make_golden as mg
  import scenes
  ref = mg.import_reference()
  from ibrnet import feature_network as ref_fn
  torch.set_grad_enabled(False)
  fx = {}

  cfg = dict(scenes.GOLDEN_CONFIGS["mv_small"], **MV77)
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  mref = mg.reference_model(ref, model, args, False)
  want = ref.rr.render_rays_mv(frame, t, offs, batch, mref, ref.proj.Projector("cpu"), feat_c, feat_f,
                               cfg["N_samples"], args, inv_uniform=True, N_importance=cfg["N_importance"],
                               det=True, is_train=False)
  fx["mv77"] = {k: mg.clean(want[k]) for k in ("outputs_coarse_ref", "outputs_fine_ref", "outputs_fine_ref_dy")}
  fx["mv77"]["checksum"] = mg.checksum(batch, [feat_c, feat_f])

  cfg = dict(scenes.GOLDEN_CONFIGS["mv_small"], **SAMPLER91)
  batch = scenes.build(cfg)[0]
  data = scenes.sampler_data(batch, cfg["H"], cfg["W"], cfg["seed"])
  fx["sampler91"] = {}
  for stride in (1, 3):
    got = ref.sr.RaySamplerSingleImage(data, "cpu", render_stride=stride).get_all()
    fx["sampler91"][stride] = {k: (v.clone() if torch.is_tensor(v) else None) for k, v in got.items()}

  args = checkpoint_args()
  torch.manual_seed(3)
  mods = {"net_fine_st": ref.mlp.DynibarStatic(args, 32, 32), "net_fine_dy": ref.mlp.DynibarDynamic(args, 32, 32),
          "motion_mlp_fine": ref.mlp.MotionMLP(num_basis=6)}
  fx["ckpt"] = {k: [(n, tuple(v.shape)) for n, v in m.state_dict().items()] for k, m in mods.items()}

  fx["encoder"] = {}
  for N, H, W in ENCODER_SHAPES:
    r = scenes.encoder_weights(ref_fn.ResNet(coarse_out_ch=32, fine_out_ch=32, coarse_only=False), N * 1000 + H)
    x = encoder_input(N, H, W)
    wc, wf = r.eval()(x)
    idx = encoder_sample(wc.numel(), N, H)
    fx["encoder"][(N, H, W)] = dict(shape=tuple(wc.shape), input_sum=float(x.double().sum()),
                                    coarse=wc.flatten()[idx].clone(), fine=wf.flatten()[idx].clone())

  path = os.path.join(HERE, "live_reference.pt")
  torch.save(fx, path)
  print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
  main()
