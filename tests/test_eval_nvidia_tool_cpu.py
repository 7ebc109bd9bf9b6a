"""tools/eval_nvidia.py's printed lines, with the scene, the model and the weights stubbed: the reference's 9 MOVING
lines per time step and 9 AVG lines in its order (eval_nvidia.py:459-481) with --lpips_alexnet / --lpips_lin, and
the 6 + 6 lines of PSNR and SSIM alone without them."""

import contextlib
import importlib.util
import io
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LABELS = ["PSNR", "SSIM", "LPIPS", "DYNAMIC PSNR", "DYNAMIC SSIM", "DYNAMIC LPIPS", "Static PSNR", "Static SSIM",
              "Static LPIPS"]
T = 3


def _tool():
  spec = importlib.util.spec_from_file_location("eval_nvidia_tool", os.path.join(ROOT, "tools", "eval_nvidia.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


class _Scene(object):
  num_frames = T + 6

  def __init__(self, path, args, dev):
    pass

  def evaluate(self, model, projector, args, on_step=None, lpips=None):
    rng = np.random.default_rng(0)
    scores, lp = rng.random((T, 11, 3, 2)), rng.random((T, 11, 3))
    for t in range(T):
      if lpips is None:
        on_step(t + 3, scores[:t + 1])
      else:
        on_step(t + 3, scores[:t + 1], lp[:t + 1])
    from dynibar_b200.nvidia_scene import mean_lpips, mean_scores
    res = dict(scores=scores, mean=mean_scores(scores), steps=list(range(3, T + 3)))
    if lpips is not None:
      res.update(lpips=lp, lpips_mean=mean_lpips(lp))
    return res


class _Enc(object):
  def to(self, dev):
    return self

  def load_state_dict(self, sd):
    pass

  def eval(self):
    return self

  def requires_grad_(self, flag):
    return self


def _run(monkeypatch, extra):
  from dynibar_b200 import feature_network, metrics, model, nvidia_scene
  monkeypatch.setattr(nvidia_scene, "NvidiaScene", _Scene)
  monkeypatch.setattr(model, "model_from_checkpoints",
                      lambda args, **kw: (type("M", (), {})(), dict(encoders=dict(feature_net={}, feature_net_fine={}))))
  monkeypatch.setattr(feature_network, "ResNet", _Enc)
  monkeypatch.setattr(metrics, "LPIPSWeights", lambda a, l, device=None: ("weights", a, l))
  buf = io.StringIO()
  with contextlib.redirect_stdout(buf):
    res = _tool().main(["--scene_path", "s", "--coarse", "c", "--fine", "f", "--device", "cpu"] + extra)
  return buf.getvalue().splitlines(), res


def _labels(lines, prefix):
  return [re.match(r"%s (.*?) +\S+$" % prefix, l).group(1) for l in lines if l.startswith(prefix + " ")]


def test_lpips_lines_in_the_reference_order(monkeypatch):
  lines, res = _run(monkeypatch, ["--lpips_alexnet", "a.pth", "--lpips_lin", "l.pth"])
  assert _labels(lines, "MOVING") == REF_LABELS * T
  assert _labels(lines, "AVG") == REF_LABELS
  avg = [l for l in lines if l.startswith("AVG ")]
  assert avg[2] == "AVG LPIPS  %s" % res["lpips_mean"][0]
  assert avg[8] == "AVG Static LPIPS  %s" % res["lpips_mean"][2]
  assert avg[0] == "AVG PSNR  %s" % res["mean"][0, 0]


def test_without_lpips_flags_the_lines_are_psnr_and_ssim(monkeypatch):
  lines, res = _run(monkeypatch, [])
  six = [l for l in REF_LABELS if "LPIPS" not in l]
  assert _labels(lines, "MOVING") == six * T
  assert lines[-6:] == ["AVG %s  %s" % (label, res["mean"][r, c]) for label, r, c in _tool().LABELS]
  assert "lpips" not in res


def test_lpips_flags_go_together(monkeypatch, capsys):
  with pytest.raises(SystemExit):
    _run(monkeypatch, ["--lpips_alexnet", "a.pth"])
  assert "go together" in capsys.readouterr().err
