"""Recipe for oracle/_ref: the UNMODIFIED reference, compiled where its sources lie.

    python oracle/build_ref.py          (also run by __graft_entry__.build() in the build container)

The reference's hot path is pure Python (ibrnet/*.py, no C/C++/CUDA).  Each module on the path is
byte-compiled from /root/reference/ibrnet/<m>.py into oracle/_ref/ibrnet/<m>.pyc -- a binary build
artefact (git-ignored, shipped to the GPU box with the snapshot, same interpreter in the same image);
no reference SOURCE is copied into this repository.  `load()` imports those sourceless modules
(plus a 4-line stand-in for kornia.create_meshgrid, which sample_ray.py imports and the image lacks).

Test / bench infrastructure only: imported by bench.py's `--impl reference` / `cpu_baseline` legs and
by tests; never by the product (dynibar_b200/)."""

import os
import py_compile
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.path.join(os.environ.get("DYNIBAR_REFERENCE", "/root/reference"), "ibrnet")
OUT = os.path.join(HERE, "_ref", "ibrnet")
MODULES = ("render_ray", "projection", "mlp_network", "render_image", "sample_ray", "feature_network")


def build():
  """Returns True when oracle/_ref was (re)built, False when /root/reference is absent."""
  if not os.path.isdir(REF_SRC):
    return False
  os.makedirs(OUT, exist_ok=True)
  for m in MODULES:
    py_compile.compile(os.path.join(REF_SRC, m + ".py"), cfile=os.path.join(OUT, m + ".pyc"),
                       dfile="ibrnet/%s.py" % m, doraise=True)
  return True


def available():
  return all(os.path.exists(os.path.join(OUT, m + ".pyc")) for m in MODULES)


def load():
  """Import the compiled reference modules -> namespace(rr, proj, mlp, ri, sr, fn)."""
  if not available():
    raise ImportError("oracle/_ref is not built (python oracle/build_ref.py in the build container)")
  root = os.path.dirname(OUT)
  if root not in sys.path:
    sys.path.insert(0, root)
  if "kornia" not in sys.modules:  # only create_meshgrid is used (sample_ray.py:6,83)
    import torch
    k = types.ModuleType("kornia")

    def create_meshgrid(H, W, normalized_coordinates=False):
      ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32),
                              indexing="ij")
      return torch.stack([xs, ys], -1)[None]

    k.create_meshgrid = create_meshgrid
    sys.modules["kornia"] = k
  import importlib
  import torch.jit._state as jit_state
  # mlp_network.py:115 decorates fused_mean_variance with @torch.jit.script, and TorchScript needs the
  # SOURCE text; with scripting switched off while importing, the decorator returns the plain Python
  # function (same arithmetic)
  was_enabled = jit_state._enabled.enabled
  jit_state.disable()
  try:
    mods = {m: importlib.import_module("ibrnet." + m) for m in MODULES}
  finally:
    if was_enabled:
      jit_state.enable()
  return types.SimpleNamespace(rr=mods["render_ray"], proj=mods["projection"], mlp=mods["mlp_network"],
                               ri=mods["render_image"], sr=mods["sample_ray"], fn=mods["feature_network"])


def reference_model(ref, model, args):
  """The reference's own nn.Modules carrying the weights of our mirror containers (strict load)."""
  import torch
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


if __name__ == "__main__":
  print("oracle/_ref built" if build() else "/root/reference not present: nothing built")
