"""tests/golden/loss_terms.pt: outputs of the reference's own loss helpers -- utils.img2charbonier and the four
callables of ibrnet/criterion.py (Criterion, compute_rgb_loss, compute_temporal_rgb_loss, compute_flow_loss) -- on
seeded inputs (run where the reference is, as make_golden.py):

    python tests/golden/make_golden_loss.py

The rest of the reference's criterion is written inline in train() (train.py:300-456) and calls a package that is not
available here, so it cannot be executed; tests/loss_ref.py says how those terms are pinned.  The reference's utils.py
imports cv2 and matplotlib for its plotting helpers only: absent ones are replaced by empty stand-in modules.
"""

import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("DYNIBAR_REFERENCE", "/root/reference")

CASES = {"a": dict(R=37, n_flow=6, seed=21), "b": dict(R=5, n_flow=3, seed=22)}


def inputs(R, n_flow, seed):
  """Seeded stand-ins for the tensors the helpers read (float32, as in training)."""
  g = torch.Generator().manual_seed(seed)
  rnd = lambda *s: torch.rand(*s, generator=g)
  outputs = {"rgb": rnd(R, 3), "mask": rnd(R) > 0.25, "occ_weight_map": rnd(R)}
  ray_batch = {"rgb": rnd(R, 3)}
  return dict(outputs=outputs, ray_batch=ray_batch, motion_mask=(rnd(R) > 0.5).float(),
              pred_mask=rnd(R) * (rnd(R) > 0.3).float(),
              render_flow=torch.randn(n_flow, R, 2, generator=g), gt_flow=torch.randn(n_flow, R, 2, generator=g),
              flow_mask=(rnd(n_flow, R, 1) > 0.3).float())


def import_reference_criterion():
  if REF not in sys.path:
    sys.path.insert(0, REF)
  for name in ("cv2", "matplotlib", "matplotlib.cm", "matplotlib.backends", "matplotlib.backends.backend_agg",
               "matplotlib.figure"):
    try:
      __import__(name)
    except ImportError:
      sys.modules[name] = types.ModuleType(name)
  sys.modules["matplotlib"].cm = sys.modules["matplotlib.cm"]
  for mod, attr in (("matplotlib.backends.backend_agg", "FigureCanvasAgg"), ("matplotlib.figure", "Figure")):
    if not hasattr(sys.modules[mod], attr):
      setattr(sys.modules[mod], attr, None)
  from ibrnet import criterion
  return criterion


def main():
  crit = import_reference_criterion()
  torch.set_grad_enabled(False)
  fx = {}
  for name, cfg in CASES.items():
    x = inputs(**cfg)
    o, rb, mm = x["outputs"], x["ray_batch"], x["motion_mask"]
    fx[name] = {
        "input_sum": float(sum(v.double().sum() for v in (o["rgb"], rb["rgb"], x["render_flow"], x["pred_mask"]))),
        "criterion": crit.Criterion()(o, rb), "criterion_motion": crit.Criterion()(o, rb, motion_mask=mm),
        "rgb": crit.compute_rgb_loss(o["rgb"], rb, x["pred_mask"]),
        "temporal": crit.compute_temporal_rgb_loss(o, rb), "temporal_motion": crit.compute_temporal_rgb_loss(o, rb, mm),
        "flow": crit.compute_flow_loss(x["render_flow"], x["gt_flow"], x["flow_mask"]),
    }
  path = os.path.join(HERE, "loss_terms.pt")
  torch.save(fx, path)
  print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
  main()
