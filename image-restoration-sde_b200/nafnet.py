"""``ConditionalNAFNet`` (Refusion's score network) with the reference's constructor, ``forward(inp, cond, time)``
signature and state-dict names/shapes (codes/config/deraining/models/modules/DenoisingNAFNet_arch.py:87-188; latent
variant codes/config/latent-dehazing/models/modules/DenoisingNAFNet_arch.py:147-181), executed by the native library.
``DenoisingNAFNet`` is the denoising-sde task's class of the same name, ``forward(x, time)``
(codes/config/denoising-sde/models/modules/DenoisingNAFNet_arch.py:103,147-150).
"""
import ctypes

import torch
import torch.nn as nn

from . import _lib
from .unet import ConditionalUNet, _Node


def nafnet_param_shapes(img_channel, width, middle_blk_num, enc_blk_nums, dec_blk_nums, variant="conditional"):
    """State-dict entries in the reference's registration order (DenoisingNAFNet_arch.py:15-49,89-143).  The
    ``"denoising"`` variant's intro conv reads img_channel channels instead of 2 * img_channel."""
    S = {}
    td = width * 4
    S["time_mlp.1.weight"] = (td * 2, width)
    S["time_mlp.1.bias"] = (td * 2,)
    S["time_mlp.3.weight"] = (td, td)
    S["time_mlp.3.bias"] = (td,)
    S["intro.weight"] = (width, img_channel * 2 if variant == "conditional" else img_channel, 3, 3)
    S["intro.bias"] = (width,)
    S["ending.weight"] = (img_channel, width, 3, 3)
    S["ending.bias"] = (img_channel,)

    def blk(pre, c):
        S[pre + "beta"] = (1, c, 1, 1)
        S[pre + "gamma"] = (1, c, 1, 1)
        S[pre + "mlp.1.weight"] = (4 * c, td // 2)
        S[pre + "mlp.1.bias"] = (4 * c,)
        for name, shp in (("conv1", (2 * c, c, 1, 1)), ("conv2", (2 * c, 1, 3, 3)), ("conv3", (c, c, 1, 1)),
                          ("sca.1", (c, c, 1, 1)), ("conv4", (2 * c, c, 1, 1)), ("conv5", (c, c, 1, 1))):
            S[pre + name + ".weight"] = shp
            S[pre + name + ".bias"] = (shp[0],)
        S[pre + "norm1.g"] = (1, c, 1, 1)
        S[pre + "norm2.g"] = (1, c, 1, 1)

    chan = width
    for i, num in enumerate(enc_blk_nums):
        for j in range(num):
            blk("encoders.%d.%d." % (i, j), chan)
        chan *= 2
    mid_c = chan
    for i, num in enumerate(dec_blk_nums):
        chan //= 2
        for j in range(num):
            blk("decoders.%d.%d." % (i, j), chan)
    for j in range(middle_blk_num):
        blk("middle_blks.%d." % j, mid_c)
    chan = mid_c
    for i in range(len(dec_blk_nums)):
        S["ups.%d.0.weight" % i] = (chan * 2, chan, 1, 1)
        chan //= 2
    chan = width
    for i in range(len(enc_blk_nums)):
        S["downs.%d.weight" % i] = (chan * 2, chan, 2, 2)
        S["downs.%d.bias" % i] = (chan * 2,)
        chan *= 2
    return S


def infer_nafnet_config(state_dict):
    """(img_channel, width, middle_blk_num, enc_blk_nums, dec_blk_nums, variant) of a ConditionalNAFNet state dict in the
    reference's naming, or None.  Only an exact match with ``nafnet_param_shapes`` (same keys in the same order, same
    shapes) is accepted, so networks with extra modules (stereo-sr's ``fusion.*``, latent-bokeh's ``cam_mlp.*``) decline.
    The image-space and latent forms have identical state dicts; ``shadow.adopt`` tells them apart by a probe."""
    try:
        sd = state_dict
        width, cin = sd["intro.weight"].shape[:2]
        img_channel = sd["ending.weight"].shape[0]
        variant = {img_channel: "denoising", 2 * img_channel: "conditional"}.get(cin)
        if variant is None:
            return None

        def blocks(prefix):   # number of blocks j with keys "<prefix>j."
            js = [int(k[len(prefix):].split(".")[0]) for k in sd if k.startswith(prefix)]
            return max(js) + 1 if js else 0

        enc = [blocks("encoders.%d." % i) for i in range(len([k for k in sd if k.startswith("downs.") and k.endswith(".weight")]))]
        dec = [blocks("decoders.%d." % i) for i in range(len([k for k in sd if k.startswith("ups.")]))]
        middle = blocks("middle_blks.")
        if len(enc) != len(dec) or len(enc) > 8:
            return None
        shapes = nafnet_param_shapes(img_channel, width, middle, enc, dec, variant)
        if list(shapes) != list(sd) or any(tuple(sd[k].shape) != tuple(v) for k, v in shapes.items()):
            return None
        return img_channel, width, middle, enc, dec, variant
    except Exception:
        return None


class _NafConfig(ctypes.Structure):
    _fields_ = [("img_channel", ctypes.c_int32), ("width", ctypes.c_int32), ("middle_blk_num", ctypes.c_int32),
                ("n_levels", ctypes.c_int32), ("enc_blk_nums", ctypes.c_int32 * 8), ("dec_blk_nums", ctypes.c_int32 * 8),
                ("latent", ctypes.c_int32), ("precision", ctypes.c_int32), ("device", ctypes.c_int32),
                ("flags", ctypes.c_int32)]


class _NafContext(_lib.Context):
    def __init__(self, img_channel, width, middle, enc, dec, latent, precision, device_index, force_simt=False,
                 variant=_lib.NET_CONDITIONAL):
        L = _lib.load()
        L.irsde_create_nafnet_variant.argtypes = [ctypes.POINTER(_NafConfig), ctypes.c_int32, ctypes.POINTER(ctypes.c_void_p)]
        L.irsde_create_nafnet_variant.restype = ctypes.c_int
        cfg = _NafConfig(img_channel, width, middle, len(enc), (ctypes.c_int32 * 8)(*enc), (ctypes.c_int32 * 8)(*dec),
                         1 if latent else 0, precision, device_index, 1 if force_simt else 0)
        h = ctypes.c_void_p()
        _lib.check(L.irsde_create_nafnet_variant(ctypes.byref(cfg), variant, ctypes.byref(h)))
        self.h = h
        self.L = L


class ConditionalNAFNet(ConditionalUNet):
    """Drop-in for the reference ``ConditionalNAFNet``.  ``latent=True`` selects the latent-dehazing variant
    (``ending(x + intro(x))``).  Inherits weight upload / forward plumbing from ``ConditionalUNet``."""

    variant = "conditional"

    def __init__(self, img_channel=3, width=16, middle_blk_num=1, enc_blk_nums=[], dec_blk_nums=[], upscale=1,
                 latent=False, precision=None, force_simt=False):
        nn.Module.__init__(self)
        import os
        if len(enc_blk_nums) != len(dec_blk_nums) or len(enc_blk_nums) > 8:
            raise ValueError("enc_blk_nums / dec_blk_nums must have the same length (<= 8)")
        self.in_nc = self.out_nc = img_channel
        self.img_channel, self.width, self.middle_blk_num = img_channel, width, middle_blk_num
        self.enc_blk_nums, self.dec_blk_nums = list(enc_blk_nums), list(dec_blk_nums)
        self.upscale, self.latent = upscale, latent
        self.precision = precision or os.environ.get("IRSDE_B200_PRECISION", "fp32")
        if self.precision not in _lib.PRECISIONS:
            raise ValueError("precision must be one of %s" % (sorted(_lib.PRECISIONS),))
        self._force_simt = force_simt
        self._shapes = nafnet_param_shapes(img_channel, width, middle_blk_num, enc_blk_nums, dec_blk_nums, self.variant)
        for name, shp in self._shapes.items():
            parts = name.split(".")
            node = self
            for p in parts[:-1]:
                if p not in node._modules:
                    node.add_module(p, _Node())
                node = node._modules[p]
            if name.endswith("beta") or name.endswith("gamma"):
                init = torch.zeros(shp)  # reference: zeros (DenoisingNAFNet_arch.py:45-46)
            else:
                init = self._init(name, shp)
            node.register_parameter(parts[-1], nn.Parameter(init))
        self._ctx = None
        self._ctx_dev = None
        self._sig = None

    def _context(self, device):
        if device.type != "cuda":
            raise RuntimeError("irsde_b200.ConditionalNAFNet runs on CUDA (sm_90a) only; there is no CPU path")
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if self._ctx is None or self._ctx_dev != idx:
            if self._ctx is not None:
                self._ctx.close()
            self._ctx = _NafContext(self.img_channel, self.width, self.middle_blk_num, self.enc_blk_nums, self.dec_blk_nums,
                                    self.latent, _lib.PRECISIONS[self.precision], idx, force_simt=self._force_simt,
                                    variant=_lib.NET_CONDITIONAL if self.variant == "conditional" else _lib.NET_DENOISING)
            self._ctx_dev = idx
            self._sig = None
        return self._ctx

    @torch.no_grad()
    def forward(self, inp, cond, time):
        return self._run(inp, cond, time)


class DenoisingNAFNet(ConditionalNAFNet):
    """The denoising-sde task's ``ConditionalNAFNet``: no condition input, intro conv over the img_channel channels of x
    (codes/config/denoising-sde/models/modules/DenoisingNAFNet_arch.py:87-150).  Drives ``DenoisingSDE``."""

    variant = "denoising"

    def __init__(self, img_channel=3, width=16, middle_blk_num=1, enc_blk_nums=[], dec_blk_nums=[], upscale=1,
                 precision=None, force_simt=False):
        super().__init__(img_channel, width, middle_blk_num, enc_blk_nums, dec_blk_nums, upscale, False, precision,
                         force_simt)

    @torch.no_grad()
    def forward(self, x, time):
        return self._run(x, None, time)
