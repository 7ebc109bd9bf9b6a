"""The virtual-source-view kernels (csrc/splat.cu, dynibar_b200.virtual_views) on the GPU against the float64
restatement (tests/virtual_views_ref.py) and against the PNGs the unmodified reference script wrote
(tests/golden/virtual_views.pt).  Bars: tests/virtual_views_ref.py BARS / PNG_FRAC_BAR, stated in DESIGN §3.5.
Every entry point is also run twice and must give the same bits."""

import numpy as np
import pytest
import torch

import virtual_views_ref as vr
from dynibar_b200 import _lib
from dynibar_b200 import virtual_views as vv

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _report(name, value):
  print("\n[virtual_views] %s = %.3e" % (name, value), end="")


@pytest.mark.parametrize("case", ["odd", "edges", "pileup", "batch"])
def test_splat_matches_restatement(case):
  frame, flow, metric = vr.splat_case(case)
  got = vv.splatting_function("softmax", frame.to(DEV), flow.to(DEV), metric.to(DEV))
  err = vr.max_err(got, vr.splat64(frame, flow, metric))
  _report("splat[%s] max abs err" % case, err)
  assert err <= vr.BARS["splat"], err
  if case == "edges":  # targets no source reaches are 0, not NaN
    assert torch.isfinite(got).all()


@pytest.mark.parametrize("case", ["batch", "const"])
def test_forward_splat_matches_restatement(case):
  imgs, d, r, t, k = vr.forward_case(case)
  img, disp = vv.render_forward_splat(imgs.to(DEV), d.to(DEV), r, t, k, k)
  want_img, want_disp = vr.render_forward_splat64(imgs, d, r, t, k, k)
  e_img, e_disp = vr.max_err(img, want_img), vr.max_err(disp, want_disp)
  _report("forward_splat[%s] image max abs err" % case, e_img)
  _report("forward_splat[%s] disp max abs err" % case, e_disp)
  assert img.shape == imgs.permute(0, 3, 1, 2).shape and disp.shape == d[:, None].shape
  assert e_img <= vr.BARS["forward_image"] and e_disp <= vr.BARS["forward_disp"], (e_img, e_disp)


@pytest.mark.parametrize("beta", [0.5, 10.0])
def test_sobel_matches_restatement(beta):
  x = vr.sobel_case()
  got = vv.sobel_fg_alpha(x[:, None].to(DEV), "sobel", beta=beta)
  err = vr.max_err(got[:, 0], vr.sobel_alpha64(x, beta))
  _report("sobel[beta=%g] max abs err" % beta, err)
  assert err <= vr.BARS["sobel"], err


def test_virtual_views_match_restatement():
  img, disp, K, ref2w, tgt = vr.frame_case()
  got = vv.render_virtual_views(torch.from_numpy(img).to(DEV), torch.from_numpy(disp).to(DEV), K, ref2w, tgt)
  want = vr.views64(img, disp, K, ref2w, tgt)
  frac = vr.png_mismatch(got.cpu().numpy(), want)
  _report("virtual_views[288x512] share of bytes > 1 LSB off", frac)
  assert got.dtype == torch.uint8 and tuple(got.shape) == want.shape
  assert frac <= vr.PNG_FRAC_BAR, frac


@pytest.mark.parametrize("i", [0, 1])
def test_virtual_views_match_reference_pngs(golden, i):
  fx = golden("virtual_views")
  img, disp, K, ref2w, tgt = vr.fixture_frame_inputs(fx, i)
  got = vv.render_virtual_views(img.to(DEV), disp.to(DEV), K, ref2w, tgt).cpu().numpy()
  frac = vr.png_mismatch(got, vr.decode_pngs(fx["frames"][i]["png"]))
  _report("virtual_views[fixture %d] share of bytes > 1 LSB off" % i, frac)
  assert frac <= vr.PNG_FRAC_FIXTURE_BAR, frac


def test_bit_identical_repeats():
  frame, flow, metric = (a.to(DEV) for a in vr.splat_case("pileup"))
  a = vv.splatting_function("softmax", frame, flow, metric)
  assert torch.equal(a, vv.splatting_function("softmax", frame, flow, metric))
  imgs, d, r, t, k = vr.forward_case("batch")
  a = vv.render_forward_splat(imgs.to(DEV), d.to(DEV), r, t, k, k)
  b = vv.render_forward_splat(imgs.to(DEV), d.to(DEV), r, t, k, k)
  assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
  x = vr.sobel_case()[:, None].to(DEV)
  assert torch.equal(vv.sobel_fg_alpha(x, beta=0.5), vv.sobel_fg_alpha(x, beta=0.5))
  img, disp, K, ref2w, tgt = vr.frame_case()
  img, disp = torch.from_numpy(img).to(DEV), torch.from_numpy(disp).to(DEV)
  assert torch.equal(vv.render_virtual_views(img, disp, K, ref2w, tgt), vv.render_virtual_views(img, disp, K, ref2w, tgt))


def test_argument_errors():
  frame, flow, metric = (a.to(DEV) for a in vr.splat_case("odd"))
  with pytest.raises(RuntimeError, match="argument check failed"):
    vv.splatting_function("softmax", torch.zeros(1, 9, 8, 8, device=DEV), torch.zeros(1, 2, 8, 8, device=DEV),
                          torch.zeros(1, 1, 8, 8, device=DEV))
  with pytest.raises(ValueError):
    vv.splatting_function("softmax", frame, flow[:, :1], metric)
  B, C, H, W = frame.shape
  ws = torch.empty(16, dtype=torch.uint8, device=DEV)
  out = torch.empty_like(frame)
  rc = _lib.lib.dyn_splat_softmax(frame.data_ptr(), flow.data_ptr(), metric.data_ptr(), B, C, H, W, out.data_ptr(),
                                  ws.data_ptr(), ws.numel(), _lib.stream())
  assert rc == -3 and b"workspace" in _lib.lib.dyn_last_error()
  assert _lib.lib.dyn_virtual_views_workspace_bytes(8, 288, 512) > _lib.lib.dyn_splat_workspace_bytes(8, 288, 512) > 0
  with pytest.raises(RuntimeError, match="no CPU fallback"):
    vv.render_virtual_views(torch.zeros(4, 4, 3), torch.ones(4, 4, device=DEV), np.eye(3), np.eye(4),
                            np.zeros((1, 3, 4)))


def test_tool_writes_the_reference_files(golden, tmp_path, monkeypatch):
  """tools/make_virtual_views.py on the fixture's scene (regenerated from its seed) writes source_vv_poses.npy and
  the PNGs in the reference's places, equal to what the reference wrote."""
  import os
  import runpy
  import sys
  from golden import make_golden_vv as mk
  fx = golden("virtual_views")
  data, cvd = mk.write_scene(str(tmp_path), np.random.default_rng(mk.SEED))
  tool = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "make_virtual_views.py")
  monkeypatch.setattr(sys, "argv", [tool, "--data_dir", data, "--cvd_dir", cvd, "--device", DEV])
  runpy.run_path(tool, run_name="__main__")
  dense = os.path.join(data, "dense")
  assert np.array_equal(np.load(os.path.join(dense, "source_vv_poses.npy")), fx["poses"].numpy())
  from PIL import Image
  H, W = fx["final_hw"]
  for i, f in enumerate(fx["frames"]):
    got = np.stack([np.asarray(Image.open(os.path.join(dense, "source_virtual_views_%dx%d" % (W, H), "%05d" % i,
                                                       "%02d.png" % k))) for k in range(len(f["png"]))])
    assert vr.png_mismatch(got, vr.decode_pngs(f["png"])) <= vr.PNG_FRAC_FIXTURE_BAR
