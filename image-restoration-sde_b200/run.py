"""Drop-in launcher: run an UNMODIFIED reference script (codes/config/<task>/test.py, inference.py, train.py, ...)
on top of the H100-native sampler.

    python -m irsde_b200.run /path/to/codes/config/deraining/test.py -opt=options/test/ir-sde.yml
    python -m irsde_b200.run /path/to/codes/config/deraining/train.py -opt=options/train/refusion.yml

What it does before handing control to the script (nothing in the reference tree is edited):
  * chdir to the script's directory and reproduce its sys.path set-up (test.py:15-18 imports the
    cwd-local ``models``/``options`` and does ``sys.path.insert(0, "../../"); import utils``);
  * import the reference's ``utils`` package and swap ``IRSDE`` / ``DenoisingSDE`` for ours
    (codes/utils/sde_utils.py:80,373) - every other helper (img/file/deg utils) stays the reference's;
  * every script but ``train.py``: import the task's ``models.modules`` and swap ``ConditionalUNet`` and
    ``ConditionalNAFNet`` for ours (the factory is ``getattr(M, which_model_G)(**setting)``, models/networks.py:10-15),
    choosing the variant by the reference class's own ``forward`` signature (``(x, time)`` => denoising-sde variant),
    and ``UNet`` (the latent autoencoder) too;
  * ``train.py``: keep the reference's network classes, which autograd trains; validation sampling (train.py:261-281)
    runs the module on the native kernels through a shadow the sampler adopts while the module is in eval mode
    (``irsde_b200.adopt``).  Only the frozen autoencoder ``networks.define_L`` builds (latent-dehazing's
    ``network_L: UNet``) becomes ``irsde_b200.UNet``: its ``encode`` / ``decode`` run natively in the train loop and in
    validation;
  * provide tiny stand-ins for optional third-party modules the scripts import but this image lacks
    (IPython.embed, lpips.LPIPS, lmdb, ema_pytorch.EMA, timm's layers for the DiT module that latent-dehazing's
    ``models.modules`` imports) - only when the real ones are not importable.

Precision / graph / RNG / adoption knobs come from the environment so existing YAMLs still parse:
IRSDE_B200_PRECISION=fp32|bf16|fp32x3, IRSDE_B200_GRAPH=0|1, IRSDE_B200_RNG=torch|philox, IRSDE_B200_ADOPT=0|1.

Two launcher options (before the script path) exist for A/B parity runs (tests/test_gpu_dropin.py,
tests/test_gpu_train_dropin.py):
  --seed N       torch.manual_seed(N) right before the script starts (test.py never seeds: noise_state and the per-step
                 randn_like draws are otherwise irreproducible; train.py's own seeding is commented out, train.py:75);
  --reference    do NOT swap anything: only the stand-ins for missing optional modules and the seed, i.e. the unmodified
                 reference on its own PyTorch path - the other arm of the comparison.
"""
import importlib
import inspect
import os
import runpy
import sys
import types


def _stub_missing():
    def have(name):
        try:
            importlib.import_module(name)
            return True
        except Exception:
            return False

    if not have("IPython"):
        m = types.ModuleType("IPython")
        m.embed = lambda *a, **k: None
        sys.modules["IPython"] = m
    if not have("lpips"):
        import torch

        class LPIPS(torch.nn.Module):  # metric only; needs AlexNet weights from the network
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
        import torch

        class EMA(torch.nn.Module):
            def __init__(self, model, **kw):
                super().__init__()
                self.ema_model = model

            def update(self):
                pass

        m = types.ModuleType("ema_pytorch")
        m.EMA = EMA
        sys.modules["ema_pytorch"] = m
    if not have("timm"):
        # latent-dehazing's models/modules/__init__.py imports DiT_arch, which needs these names; no shipped config
        # builds a DiT, so the stand-ins only have to import
        def unavailable(*a, **k):
            raise ImportError("timm is not installed: the DiT networks need it")

        def to_2tuple(x):
            return tuple(x) if isinstance(x, (list, tuple)) else (x, x)

        vit, layers = types.ModuleType("timm.models.vision_transformer"), types.ModuleType("timm.models.layers")
        vit.Attention = vit.Mlp = unavailable
        layers.to_2tuple = to_2tuple
        models = types.ModuleType("timm.models")
        models.vision_transformer, models.layers = vit, layers
        timm = types.ModuleType("timm")
        timm.models = models
        sys.modules.update({"timm": timm, "timm.models": models, "timm.models.vision_transformer": vit,
                            "timm.models.layers": layers})


def install(script_dir, train=False):
    """Patch the reference packages reachable from ``script_dir`` (idempotent).  ``train``: the script is the task's
    ``train.py`` - swap the samplers and the frozen autoencoder only."""
    import irsde_b200
    codes = os.path.abspath(os.path.join(script_dir, "..", ".."))
    for p in (script_dir, codes):
        if p not in sys.path:
            sys.path.insert(0, p)
    _stub_missing()
    utils = importlib.import_module("utils")
    utils.IRSDE = irsde_b200.IRSDE
    utils.DenoisingSDE = irsde_b200.DenoisingSDE
    if hasattr(utils, "sde_utils"):
        utils.sde_utils.IRSDE = irsde_b200.IRSDE
        utils.sde_utils.DenoisingSDE = irsde_b200.DenoisingSDE
    mods = importlib.import_module("models.modules")
    if train:
        networks = importlib.import_module("models.networks")
        if hasattr(networks, "define_L") and not getattr(networks.define_L, "_irsde_b200", False):
            networks.define_L = _native_define_L(networks.define_L, mods)
        return utils, mods

    def denoising(name):  # (self, x, time): the denoising-sde variant of the reference class
        ref_cls = getattr(mods, name, None)
        return ref_cls is not None and len(inspect.signature(ref_cls.forward).parameters) == 3

    mods.ConditionalUNet = irsde_b200.DenoisingUNet if denoising("ConditionalUNet") else irsde_b200.ConditionalUNet
    if hasattr(mods, "ConditionalNAFNet"):
        latent = "latent" in os.path.basename(os.path.abspath(script_dir))
        import functools
        if latent:
            mods.ConditionalNAFNet = functools.partial(irsde_b200.ConditionalNAFNet, latent=latent)
        elif denoising("ConditionalNAFNet"):
            mods.ConditionalNAFNet = irsde_b200.DenoisingNAFNet
        else:
            mods.ConditionalNAFNet = irsde_b200.ConditionalNAFNet
    if hasattr(mods, "UNet"):
        mods.UNet = irsde_b200.UNet
    return utils, mods


def _native_define_L(reference_define_L, mods):
    """``networks.define_L`` returning ``irsde_b200.UNet`` for ``network_L: UNet``.  The reference's module is still
    built first and its initial weights copied, so the global generator advances exactly as in the reference and the
    rest of the run draws the same numbers (load_network then overwrites the weights with the pretrained ones)."""
    import torch
    import irsde_b200

    def define_L(opt):
        ref = reference_define_L(opt)
        if opt["network_L"]["which_model"] != "UNet" or not isinstance(ref, mods.UNet):
            return ref
        with torch.random.fork_rng(devices=[]):
            net = irsde_b200.UNet(**opt["network_L"]["setting"])
        net.load_state_dict(ref.state_dict())
        return net

    define_L._irsde_b200 = True
    return define_L


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    seed, reference = None, False
    while argv and argv[0].startswith("--"):
        opt = argv.pop(0)
        if opt == "--seed":
            seed = int(argv.pop(0))
        elif opt == "--reference":
            reference = True
        else:
            raise SystemExit("unknown launcher option %s\n%s" % (opt, __doc__))
    if not argv:
        raise SystemExit(__doc__)
    script = os.path.abspath(argv[0])
    script_dir = os.path.dirname(script)
    os.chdir(script_dir)
    if reference:
        codes = os.path.abspath(os.path.join(script_dir, "..", ".."))
        for p in (script_dir, codes):
            if p not in sys.path:
                sys.path.insert(0, p)
        _stub_missing()
    else:
        install(script_dir, train=os.path.basename(script) == "train.py")
    if seed is not None:
        import torch
        torch.manual_seed(seed)
    sys.argv = [script] + argv[1:]
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
