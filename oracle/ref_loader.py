"""Import the staged, unmodified reference (oracle/_ref, see make_ref.py) the way its own scripts do.

`codes/config/<task>/test.py` resolves `models` / `options` from its cwd and `utils` / `data` from `../../`
(test.py:14-20); load(task) reproduces that search path and returns the reference's own modules.  Optional third-party
imports the scripts make but this image lacks (IPython, lpips, lmdb, ema_pytorch, timm) get inert stand-ins - only when
the real package is not importable.  Nothing of irsde_b200 is imported here: this is the reference arm.
"""
import importlib
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(HERE, "_ref")


def available():
    return os.path.exists(os.path.join(REF, ".staged"))


def stub_missing():
    def have(name):
        try:
            importlib.import_module(name)
            return True
        except Exception:
            return False

    import torch
    if not have("IPython"):
        m = types.ModuleType("IPython")
        m.embed = lambda *a, **k: None
        sys.modules["IPython"] = m
    if not have("lpips"):
        class LPIPS(torch.nn.Module):  # perceptual METRIC only (needs AlexNet weights from the network); not on the path
            def __init__(self, net="alex", **kw):
                super().__init__()

            def forward(self, a, b):
                return torch.zeros(1, device=a.device)

        m = types.ModuleType("lpips")
        m.LPIPS = LPIPS
        sys.modules["lpips"] = m
    if not have("lmdb"):
        sys.modules["lmdb"] = types.ModuleType("lmdb")
    if not have("ema_pytorch"):
        class EMA(torch.nn.Module):
            def __init__(self, model, **kw):
                super().__init__()
                self.ema_model = model

            def update(self):
                pass

        m = types.ModuleType("ema_pytorch")
        m.EMA = EMA
        sys.modules["ema_pytorch"] = m


def task_dir(task="deraining"):
    return os.path.join(REF, "codes", "config", task)


def load(task="deraining"):
    """-> (utils module, models.modules module) of the reference task directory."""
    if not available():
        raise ImportError("oracle/_ref is not staged (python oracle/make_ref.py needs the reference checkout)")
    td = task_dir(task)
    for p in (os.path.join(REF, "codes"), td):
        if p in sys.path:
            sys.path.remove(p)
        sys.path.insert(0, p)
    stub_missing()
    utils = importlib.import_module("utils")
    mods = importlib.import_module("models.modules")
    assert os.path.abspath(utils.__file__).startswith(REF) and os.path.abspath(mods.__file__).startswith(REF)
    return utils, mods
