"""Native shadows of foreign score networks: the reference's own PyTorch ``ConditionalUNet`` / ``ConditionalNAFNet``
(codes/config/*/models/modules/DenoisingUNet_arch.py, DenoisingNAFNet_arch.py) while ``train.py`` trains it by autograd.

A shadow keeps no weights of its own: ``sync_weights`` re-reads the foreign module's parameters whenever their
``(data_ptr, _version)`` signature changes (optimizer steps bump the versions), so validation sampling
(train.py:261-281) runs on the native kernels with the module's current weights while training stays on the
reference's autograd path.
"""
import torch

from .nafnet import ConditionalNAFNet, DenoisingNAFNet, infer_nafnet_config
from .unet import ConditionalUNet, DenoisingUNet, infer_unet_config

# The NAFNet probe: one seeded input through the foreign forward and each native form, at a mid-chain timestep.  A form
# matches when max|native - foreign| / max|foreign| is within the bound of the shadow's precision (fp32 / fp32x3 agree to
# ~1e-5 per forward, bf16 to ~1e-2); the wrong latent / image-space form is off by the size of ending(intro(x)), O(1).
PROBE_T = 50
PROBE_BOUND = {"fp32": 1e-2, "fp32x3": 1e-2, "bf16": 6e-2}


def _bind(net, module):
    for p in net.parameters():       # the shadow's own tensors are never used: do not keep a second copy of the weights
        p.data = torch.empty(0)
    net._source = module
    net.eval()
    return net


def _adopt_unet(module, sd, cfg, precision):
    in_nc, out_nc, nf, mult, variant = cfg
    plain = mult == [2 ** (i + 1) for i in range(len(mult))]
    if variant == "denoising":
        if not plain:
            return None
        net = DenoisingUNet(in_nc, out_nc, nf, depth=len(mult), precision=precision)
    else:
        net = ConditionalUNet(in_nc, out_nc, nf, depth=len(mult), precision=precision, ch_mult=None if plain else mult)
    if list(net._shapes.keys()) != list(sd.keys()) or any(tuple(sd[k].shape) != tuple(v) for k, v in net._shapes.items()):
        return None
    return _bind(net, module)


def _foreign_forward(module, x, cond, t):
    """The foreign module's own forward in eval mode without autograd; every submodule's mode is restored after."""
    modes = [(m, m.training) for m in module.modules()]
    module.eval()
    try:
        with torch.no_grad():
            return module(x, t) if cond is None else module(x, cond, t)
    finally:
        for m, mode in modes:
            m.training = mode


def _adopt_nafnet(module, cfg, precision):
    img_channel, width, middle, enc, dec, variant = cfg
    dev = next(module.parameters()).device
    if dev.type != "cuda":
        return None
    if variant == "denoising":
        forms = {"plain": DenoisingNAFNet(img_channel, width, middle, enc, dec, precision=precision)}
    else:
        forms = {name: ConditionalNAFNet(img_channel, width, middle, enc, dec, latent=latent, precision=precision)
                 for name, latent in (("plain", False), ("latent", True))}
    # the probe's input comes from a private generator: the caller's global CPU / CUDA streams stay in the reference's order
    side = max(32, 2 ** len(enc))
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, img_channel, side, side, generator=g).to(dev)
    cond = torch.rand(1, img_channel, side, side, generator=g).to(dev) if variant == "conditional" else None
    want = _foreign_forward(module, x, cond, PROBE_T).float()
    scale = want.abs().max().clamp_min(1e-12)
    errors = {}
    for name, net in forms.items():
        _bind(net, module)
        errors[name] = ((net._run(x, cond, PROBE_T) - want).abs().max() / scale).item()
    bound = PROBE_BOUND[next(iter(forms.values())).precision]
    matched = [name for name, e in errors.items() if e <= bound]
    for name, net in forms.items():
        if matched != [name] and net._ctx is not None:
            net._ctx.close()
            net._ctx = None
    if len(matched) != 1:
        return None
    net = forms[matched[0]]
    net.probe_errors, net.probe_bound = errors, bound
    return net


def adopt(module, precision=None):
    """Native shadow of a foreign ``nn.Module`` with the state-dict layout of the reference's ``ConditionalUNet`` (either
    task variant) or ``ConditionalNAFNet`` (the conditional, denoising-sde and latent-dehazing forms), or None.

    The latent NAFNet computes ``ending(x + intro(x))`` with the same parameters as the image-space one, so a NAFNet is
    adopted only after a probe: the module's own forward and each candidate form on one seeded input; the form within
    ``PROBE_BOUND`` wins (``probe_errors`` / ``probe_bound`` on the shadow record the evidence) and no match declines.
    Adoption leaves the module's mode, its parameters and the global random generators as it found them."""
    sd = module.state_dict()
    dev = next(module.parameters()).device if any(True for _ in module.parameters()) else torch.device("cpu")
    cuda = [dev.index if dev.index is not None else torch.cuda.current_device()] if dev.type == "cuda" else []
    with torch.random.fork_rng(devices=cuda):    # the native constructors draw their (unused) initial weights
        cfg = infer_unet_config(sd)
        if cfg is not None:
            return _adopt_unet(module, sd, cfg, precision)
        cfg = infer_nafnet_config(sd)
        if cfg is not None:
            return _adopt_nafnet(module, cfg, precision)
    return None
