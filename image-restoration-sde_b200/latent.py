"""Refusion latent autoencoder ``UNet`` with the reference's constructor and ``encode`` / ``decode`` / ``forward``
(codes/config/latent-dehazing/models/modules/UNet_arch.py:17-97), executed by the native library.

``encode(x)`` returns ``(z, h)`` like the reference; ``h`` is an opaque handle (the skip features stay in device
buffers owned by the native context and are consumed by the next ``decode(z, h)`` of the same input shape), which is
how the reference's callers use it (latent-dehazing/test.py:90, models/latent_denoising_model.py:189)."""
import ctypes

import torch
import torch.nn as nn

from . import _lib
from .unet import ConditionalUNet, _Node


def latent_unet_param_shapes(in_ch, out_ch, ch, ch_mult, embed_dim):
    """State-dict entries in the reference's registration order (UNet_arch.py:18-51)."""
    S = {}
    depth = len(ch_mult)
    m = [1] + list(ch_mult)
    S["init_conv.weight"] = (ch, in_ch, 3, 3)

    def rb(pre, ci, co):
        S[pre + "block1.proj.weight"] = (co, ci, 3, 3)
        S[pre + "block2.proj.weight"] = (co, co, 3, 3)
        if ci != co:
            S[pre + "res_conv.weight"] = (co, ci, 1, 1)

    def la(pre, c):
        S[pre + "fn.fn.to_qkv.weight"] = (384, c, 1, 1)
        S[pre + "fn.fn.to_out.0.weight"] = (c, 128, 1, 1)
        S[pre + "fn.fn.to_out.0.bias"] = (c,)
        S[pre + "fn.fn.to_out.1.g"] = (1, c, 1, 1)
        S[pre + "fn.norm.g"] = (1, c, 1, 1)

    dec = []
    for i in range(depth):
        di, do = ch * m[i], ch * m[i + 1]
        pre = "encoder.%d." % i
        rb(pre + "0.", di, di)
        rb(pre + "1.", di, di)
        if i == depth - 1:
            la(pre + "2.", di)
        if i != depth - 1:
            S[pre + "3.weight"] = (do, di, 4, 4)
            S[pre + "3.bias"] = (do,)
        else:
            S[pre + "3.weight"] = (do, di, 3, 3)
        dec.insert(0, (i, di, do))
    for j, (i, di, do) in enumerate(dec):
        pre = "decoder.%d." % j
        rb(pre + "0.", do + di, do)
        rb(pre + "1.", do + di, do)
        if i == depth - 1:
            la(pre + "2.", do)
        if i != 0:
            S[pre + "3.1.weight"] = (di, do, 3, 3)
            S[pre + "3.1.bias"] = (di,)
        else:
            S[pre + "3.weight"] = (di, do, 3, 3)
    mid = ch * m[-1]
    S["latent_conv.weight"] = (embed_dim, mid, 1, 1)
    S["post_latent_conv.weight"] = (mid, embed_dim, 1, 1)
    S["final_conv.weight"] = (out_ch, ch, 3, 3)
    S["final_conv.bias"] = (out_ch,)
    return S


class _LatConfig(ctypes.Structure):
    _fields_ = [("in_ch", ctypes.c_int32), ("out_ch", ctypes.c_int32), ("ch", ctypes.c_int32), ("n_levels", ctypes.c_int32),
                ("ch_mult", ctypes.c_int32 * 8), ("embed_dim", ctypes.c_int32), ("precision", ctypes.c_int32),
                ("device", ctypes.c_int32), ("flags", ctypes.c_int32)]


class _LatContext(_lib.Context):
    def __init__(self, in_ch, out_ch, ch, ch_mult, embed_dim, precision, device_index, force_simt=False):
        L = _lib.load()
        vp, i32 = ctypes.c_void_p, ctypes.c_int32
        L.irsde_create_latent_unet.argtypes = [ctypes.POINTER(_LatConfig), ctypes.POINTER(vp)]
        L.irsde_create_latent_unet.restype = ctypes.c_int
        L.irsde_latent_shape.argtypes = [vp, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32)]
        L.irsde_latent_shape.restype = ctypes.c_int
        for f in (L.irsde_latent_encode, L.irsde_latent_decode):
            f.argtypes = [vp, vp, vp, i32, i32, i32, vp]
            f.restype = ctypes.c_int
        cfg = _LatConfig(in_ch, out_ch, ch, len(ch_mult), (ctypes.c_int32 * 8)(*ch_mult), embed_dim, precision, device_index,
                         1 if force_simt else 0)
        h = vp()
        _lib.check(L.irsde_create_latent_unet(ctypes.byref(cfg), ctypes.byref(h)))
        self.h = h
        self.L = L


class LatentSkips:
    """Opaque stand-in for the reference's skip list ``h``: (owner module, input shape)."""

    def __init__(self, owner, shape, gen, ctx=None):
        self.owner, self.shape, self.gen, self.ctx = owner, tuple(shape), gen, ctx


class UNet(ConditionalUNet):
    """Drop-in for the reference latent ``UNet``."""

    def __init__(self, in_ch=3, out_ch=3, ch=64, ch_mult=[1, 2, 4, 4], embed_dim=4, precision=None, force_simt=False):
        nn.Module.__init__(self)
        import os
        self.in_nc, self.out_nc = in_ch, out_ch
        self.in_ch, self.out_ch, self.ch, self.ch_mult, self.embed_dim = in_ch, out_ch, ch, list(ch_mult), embed_dim
        self.depth = len(ch_mult)
        self.precision = precision or os.environ.get("IRSDE_B200_PRECISION", "fp32")
        if self.precision not in _lib.PRECISIONS:
            raise ValueError("precision must be one of %s" % (sorted(_lib.PRECISIONS),))
        self._force_simt = force_simt
        self._shapes = latent_unet_param_shapes(in_ch, out_ch, ch, ch_mult, embed_dim)
        for name, shp in self._shapes.items():
            parts = name.split(".")
            node = self
            for p in parts[:-1]:
                if p not in node._modules:
                    node.add_module(p, _Node())
                node = node._modules[p]
            node.register_parameter(parts[-1], nn.Parameter(self._init(name, shp)))
        self._ctx = None
        self._ctx_dev = None
        self._sig = None

    def _context(self, device):
        if device.type != "cuda":
            raise RuntimeError("irsde_b200.UNet runs on CUDA (sm_90a) only; there is no CPU path")
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if self._ctx is None or self._ctx_dev != idx:
            if self._ctx is not None:
                self._ctx.close()
            self._ctx = _LatContext(self.in_ch, self.out_ch, self.ch, self.ch_mult, self.embed_dim,
                                    _lib.PRECISIONS[self.precision], idx,
                                    force_simt=self._force_simt)
            self._ctx_dev = idx
            self._sig = None
        return self._ctx

    @torch.no_grad()
    def encode(self, x):
        if not x.is_cuda:
            raise RuntimeError("irsde_b200.UNet runs on CUDA (sm_90a) only; there is no CPU path")
        x = x.contiguous().float()
        B, C, H, W = x.shape
        ctx = self.sync_weights(x.device)
        lh, lw = ctypes.c_int32(), ctypes.c_int32()
        _lib.check(ctx.L.irsde_latent_shape(ctx.h, H, W, ctypes.byref(lh), ctypes.byref(lw)), ctx.h)
        z = torch.empty((B, self.embed_dim, lh.value, lw.value), device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            st = torch.cuda.current_stream().cuda_stream
            _lib.check(ctx.L.irsde_latent_encode(ctx.h, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(z.data_ptr()), B, H, W,
                                                 ctypes.c_void_p(st)), ctx.h)
        self.H, self.W = H, W
        self._gen = getattr(self, "_gen", 0) + 1
        return z, LatentSkips(self, (B, H, W), self._gen, ctx)

    @torch.no_grad()
    def decode(self, x, h):
        if not isinstance(h, LatentSkips) or h.owner is not self:
            raise ValueError("decode needs the skip handle returned by this module's encode()")
        if h.gen != getattr(self, "_gen", 0):
            raise RuntimeError("stale skip handle: a later encode() overwrote the device-resident skips "
                               "(one outstanding encode per module)")
        B, H, W = h.shape
        if not x.is_cuda:
            raise RuntimeError("irsde_b200.UNet runs on CUDA (sm_90a) only; there is no CPU path")
        x = x.contiguous().float()
        ctx = self.sync_weights(x.device)
        if ctx is not h.ctx:
            raise RuntimeError("stale skip handle: the module moved to another device since encode()")
        lh, lw = ctypes.c_int32(), ctypes.c_int32()
        _lib.check(ctx.L.irsde_latent_shape(ctx.h, H, W, ctypes.byref(lh), ctypes.byref(lw)), ctx.h)
        if tuple(x.shape) != (B, self.embed_dim, lh.value, lw.value):
            # the library reads B*embed*lat_h*lat_w floats from x: a wrong-shaped latent would be an out-of-bounds read
            raise ValueError("latent must be %s for the %s input these skips came from, got %s"
                             % ((B, self.embed_dim, lh.value, lw.value), (B, self.in_ch, H, W), tuple(x.shape)))
        out = torch.empty((B, self.out_ch, H, W), device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            st = torch.cuda.current_stream().cuda_stream
            _lib.check(ctx.L.irsde_latent_decode(ctx.h, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), B, H, W,
                                                 ctypes.c_void_p(st)), ctx.h)
        return out

    def forward(self, x):
        z, h = self.encode(x)
        return self.decode(z, h)
