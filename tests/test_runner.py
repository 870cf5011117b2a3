"""The runner shim (cfdbench_b200/runner.py) rebinding logic, exercised on a minimal stand-in of CFDBench's `src/` tree
written by the test -- the module names the shim touches (`models.base_model.AutoCfdModel`, `models.loss`,
`models.fno.fno2d.Fno2d`, and the plug-in seam `utils/autoregressive.py:10`), none of the reference's code -- and, when
__graft_entry__.build() has installed it (oracle/install_reference.py), on the reference's own tree as well.  The
reference's scripts on the real tree are run by tests/test_gpu_runner.py."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "src")

# stand-in tree: relative path -> source
STAND_IN = {
    "models/__init__.py": "",
    "models/base_model.py": (
        "from torch import nn\n\n\n"
        "class AutoCfdModel(nn.Module):\n"
        "    def __init__(self, loss_fn):\n"
        "        super().__init__()\n"
        "        self.loss_fn = loss_fn\n"),
    "models/loss.py": (
        "class _Loss:\n"
        "    def get_score_names(self):\n"
        "        return [\"mse\", \"rmse\", \"mae\", \"nmse\"]\n\n\n"
        "def loss_name_to_fn(name):\n"
        "    return _Loss()\n"),
    "models/fno/__init__.py": "",
    "models/fno/fno2d.py": "class Fno2d:  # rebound by the runner\n    pass\n",
    "utils/__init__.py": "",
    "utils/autoregressive.py": "from models.fno.fno2d import Fno2d  # noqa: F401  (the plug-in seam)\n",
}

CODE = r'''
import sys
sys.path.insert(0, %r)
from cfdbench_b200 import runner
runner.install(%r, stub_missing=True)
import models.fno.fno2d as ref
from models.base_model import AutoCfdModel
from models.loss import loss_name_to_fn
import cfdbench_b200.fno2d as ours
assert ref.Fno2d is ours.Fno2d, "seam not rebound"
loss = loss_name_to_fn("nmse")
m = ref.Fno2d(in_chan=2, out_chan=2, n_case_params=5, loss_fn=loss, num_layers=4,
              hidden_dim=32, modes1=12, modes2=12, device="cpu")
assert isinstance(m, AutoCfdModel), "must subclass the tree's AutoCfdModel (test_multistep.py:109)"
assert m.loss_fn is loss, "the tree's loss object must be kept (train_auto.py:75,93)"
assert m.loss_fn.get_score_names() == ["mse", "rmse", "mae", "nmse"]
# the factory the scripts use picks the rebound class up (utils/autoregressive.py:10,114-125)
import utils.autoregressive as ua
assert ua.Fno2d is ours.Fno2d
print("ok")
'''


def test_runner_rebinds_the_seam_and_subclasses_reference_base(tmp_path):
    src = tmp_path / "src"
    for rel, text in STAND_IN.items():
        path = src / rel
        path.parent.mkdir(parents=True, exist_ok=True)
        path.write_text(text)
    trees = [str(src)] + ([REF] if os.path.isdir(os.path.join(REF, "models", "fno")) else [])
    for tree in trees:
        out = subprocess.run([sys.executable, "-c", CODE % (ROOT, tree)], capture_output=True, text=True,
                             env={**os.environ, "PYTHONDONTWRITEBYTECODE": "1"})
        assert out.returncode == 0, (tree, out.stderr[-2000:])
        assert out.stdout.strip().endswith("ok"), (tree, out.stdout)
