"""``ConditionalUNet`` with the reference's constructor, ``forward(xt, cond, time)`` signature and
state-dict names/shapes (codes/config/deraining/models/modules/DenoisingUNet_arch.py:19-134), executed
by the native sm_90a library.  The ``nn.Module`` only holds the parameters (so ``load_state_dict``,
``.to(device)``, ``DataParallel(...)``, ``.eval()`` keep working, models/denoising_model.py:36-45,153);
all arithmetic happens in hand-written CUDA kernels behind the C ABI.  No CPU path.
"""
import math

import torch
import torch.nn as nn

from . import _lib


def unet_param_shapes(in_nc, out_nc, nf, depth, variant="conditional", ch_mult=None):
    """State-dict entries in the reference's registration order
    (DenoisingUNet_arch.py:27-76; module_util.py:125-161,185-190).  ``ch_mult`` selects the latent-task variant
    (latent-dehazing/.../DenoisingUNet_arch.py:20,51-56): level i has nf*[1,ch_mult...][i] channels."""
    mult = [1] + list(ch_mult) if ch_mult is not None else [2 ** i for i in range(depth + 1)]
    depth = len(mult) - 1
    S = {}
    td = nf * 4
    S["init_conv.weight"] = (nf, in_nc * 2 if variant == "conditional" else in_nc, 7, 7)
    S["time_mlp.1.weight"] = (td, nf)
    S["time_mlp.1.bias"] = (td,)
    S["time_mlp.3.weight"] = (td, td)
    S["time_mlp.3.bias"] = (td,)

    def rb(pre, ci, co):
        S[pre + "mlp.1.weight"] = (2 * co, td)
        S[pre + "mlp.1.bias"] = (2 * co,)
        S[pre + "block1.proj.weight"] = (co, ci, 3, 3)
        S[pre + "block2.proj.weight"] = (co, co, 3, 3)
        if ci != co:
            S[pre + "res_conv.weight"] = (co, ci, 1, 1)

    def attn(pre, c, full=False):
        S[pre + "fn.fn.to_qkv.weight"] = (384, c, 1, 1)
        if full:
            S[pre + "fn.fn.to_out.weight"] = (c, 128, 1, 1)
            S[pre + "fn.fn.to_out.bias"] = (c,)
        else:
            S[pre + "fn.fn.to_out.0.weight"] = (c, 128, 1, 1)
            S[pre + "fn.fn.to_out.0.bias"] = (c,)
            S[pre + "fn.fn.to_out.1.g"] = (1, c, 1, 1)
        S[pre + "fn.norm.g"] = (1, c, 1, 1)

    ups = []
    for i in range(depth):
        di, do = nf * mult[i], nf * mult[i + 1]
        pre = "downs.%d." % i
        rb(pre + "0.", di, di)
        rb(pre + "1.", di, di)
        attn(pre + "2.", di)
        if i != depth - 1:
            S[pre + "3.weight"] = (do, di, 4, 4)
            S[pre + "3.bias"] = (do,)
        else:
            S[pre + "3.weight"] = (do, di, 3, 3)
        ups.insert(0, (i, di, do))
    for j, (i, di, do) in enumerate(ups):
        pre = "ups.%d." % j
        rb(pre + "0.", do + di, do)
        rb(pre + "1.", do + di, do)
        attn(pre + "2.", do)
        if i != 0:
            S[pre + "3.1.weight"] = (di, do, 3, 3)
            S[pre + "3.1.bias"] = (di,)
        else:
            S[pre + "3.weight"] = (di, do, 3, 3)
    mid = nf * mult[depth]
    rb("mid_block1.", mid, mid)
    attn("mid_attn.", mid, full=(variant != "conditional"))
    rb("mid_block2.", mid, mid)
    rb("final_res_block.", 2 * nf, nf)
    S["final_conv.weight"] = (out_nc, nf, 3, 3)
    S["final_conv.bias"] = (out_nc,)
    return S


class _Node(nn.Module):
    """Anonymous container so parameters get the reference's dotted names."""


class ConditionalUNet(nn.Module):
    """Drop-in for the reference score network.  ``precision``: "fp32" (parity mode: fp32 storage and
    FMA, matches the reference to ~1e-5 per forward) or "bf16" (perf mode: wgmma bf16 MMA with fp32
    accumulation).  Default comes from ``IRSDE_B200_PRECISION`` (env) or "fp32"."""

    variant = "conditional"

    def __init__(self, in_nc, out_nc, nf, depth=4, upscale=1, precision=None, force_simt=False, ch_mult=None):
        super().__init__()
        import os
        if isinstance(depth, (list, tuple)):   # latent-task signature: ConditionalUNet(in_nc, out_nc, nf, ch_mult)
            ch_mult, depth = list(depth), len(depth)
        if ch_mult is not None:
            ch_mult = [int(m) for m in ch_mult]
            depth = len(ch_mult)
        self.ch_mult = ch_mult
        self.in_nc, self.out_nc, self.nf, self.depth, self.upscale = in_nc, out_nc, nf, depth, upscale
        self.precision = precision or os.environ.get("IRSDE_B200_PRECISION", "fp32")
        if self.precision not in _lib.PRECISIONS:
            raise ValueError("precision must be one of %s" % (sorted(_lib.PRECISIONS),))
        self._force_simt = force_simt
        self._shapes = unet_param_shapes(in_nc, out_nc, nf, depth, self.variant, ch_mult)
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

    @staticmethod
    def _init(name, shp):
        if name.endswith(".g"):
            return torch.ones(shp)
        fan_in = 1
        for d in (shp[1:] if len(shp) > 1 else shp):
            fan_in *= d
        if name.endswith("bias"):
            # torch default: U(-1/sqrt(fan_in of the matching weight)); use the vector length as a proxy
            bound = 1.0 / math.sqrt(max(fan_in, 1))
        else:
            bound = 1.0 / math.sqrt(fan_in)
        return (torch.rand(shp) * 2 - 1) * bound

    # ---- native context management -------------------------------------------------------------
    def _context(self, device):
        if device.type != "cuda":
            raise RuntimeError("irsde_b200.ConditionalUNet runs on CUDA (sm_90a) only; there is no CPU path")
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if self._ctx is None or self._ctx_dev != idx:
            if self._ctx is not None:
                self._ctx.close()
            self._ctx = _lib.Context(self.in_nc, self.out_nc, self.nf, self.depth,
                                     _lib.NET_CONDITIONAL if self.variant == "conditional" else _lib.NET_DENOISING,
                                     _lib.PRECISIONS[self.precision], idx,
                                     force_simt=self._force_simt, ch_mult=self.ch_mult)
            self._ctx_dev = idx
            self._sig = None
        return self._ctx

    def sync_weights(self, device=None):
        """Upload parameters to the native context if they changed since the last upload.  ``_source`` (set by ``shadow.adopt``)
        names another module that owns the parameters: e.g. the reference's own PyTorch ConditionalUNet while it is being
        trained by autograd - the native network then shadows it (same state-dict names) for validation sampling."""
        import ctypes
        src = getattr(self, "_source", None)
        params = dict((src if src is not None else self).named_parameters())
        dev = device or next(iter(params.values())).device
        ctx = self._context(dev)
        sig = tuple((p.data_ptr(), p._version) for p in params.values())
        if sig == self._sig:
            return ctx
        L = ctx.L
        for name, p in params.items():
            t = p.detach()
            if t.dtype != torch.float32 or not t.is_contiguous():
                t = t.float().contiguous()
            shape = (ctypes.c_int64 * t.dim())(*t.shape)
            _lib.check(L.irsde_load_tensor(ctx.h, name.encode(), ctypes.c_void_p(t.data_ptr()), t.dim(), shape), ctx.h)
        _lib.check(L.irsde_finalize_weights(ctx.h), ctx.h)
        self._sig = sig
        self._uploads = getattr(self, "_uploads", 0) + 1
        return ctx

    # ---- forward ---------------------------------------------------------------------------------
    def _times(self, time, B):
        if isinstance(time, (int, float)):
            return [float(time)]
        t = torch.as_tensor(time).reshape(-1).float().cpu().tolist()
        if len(t) not in (1, B):
            raise ValueError("time must be a scalar or a tensor of length B")
        return t

    def _run(self, x, cond, time):
        import ctypes
        if not x.is_cuda:
            raise RuntimeError("irsde_b200.ConditionalUNet runs on CUDA (sm_90a) only; there is no CPU path")
        x = x.contiguous().float()
        if cond is not None:
            cond = cond.to(x.device).contiguous().float()
            if cond.shape != x.shape:
                raise ValueError("cond must have the shape of xt")
        B, C, H, W = x.shape
        if C != self.in_nc:
            raise ValueError("expected %d input channels, got %d" % (self.in_nc, C))
        ctx = self.sync_weights(x.device)
        times = self._times(time, B)
        out = torch.empty((B, self.out_nc, H, W), device=x.device, dtype=torch.float32)
        arr = _lib.float_array(times)
        with torch.cuda.device(x.device):
            st = torch.cuda.current_stream().cuda_stream
            _lib.check(ctx.L.irsde_noise_fn(ctx.h, ctypes.c_void_p(x.data_ptr()),
                                            ctypes.c_void_p(cond.data_ptr()) if cond is not None else None, arr,
                                            len(times), ctypes.c_void_p(out.data_ptr()), B, H, W, ctypes.c_void_p(st)),
                       ctx.h)
        return out

    @torch.no_grad()
    def forward(self, xt, cond, time):
        return self._run(xt, cond, time)

    # ---- parity instrumentation (C ABI: irsde_plan_num_ops / irsde_plan_op_info / irsde_trace_forward) ------------
    def plan_ops(self, B, H, W, device=None):
        """[(label, (C, H, W) of the NHWC view the op writes or None, category)] of the launch plan for a [B,*,H,W] input."""
        import ctypes
        ctx = self.sync_weights(device)
        n = ctx.L.irsde_plan_num_ops(ctx.h, B, H, W)
        if n < 0:
            _lib.check(n, ctx.h)
        ops, buf, dims = [], ctypes.create_string_buffer(256), (ctypes.c_int32 * 4)()
        for i in range(n):
            _lib.check(ctx.L.irsde_plan_op_info(ctx.h, B, H, W, i, buf, 256, dims), ctx.h)
            ops.append((buf.value.decode(), (dims[0], dims[1], dims[2]) if dims[0] else None, dims[3]))
        return ops

    @torch.no_grad()
    def trace(self, xt, cond, time, op):
        """Output of op `op` of the forward (fp32 [B,C,H,W]); runs ops 0..op."""
        import ctypes
        x = xt.contiguous().float()
        cond = cond.to(x.device).contiguous().float() if cond is not None else None
        B, _, H, W = x.shape
        ctx = self.sync_weights(x.device)
        buf, dims = ctypes.create_string_buffer(256), (ctypes.c_int32 * 4)()
        _lib.check(ctx.L.irsde_plan_op_info(ctx.h, B, H, W, op, buf, 256, dims), ctx.h)
        out = torch.empty((B, dims[0], dims[1], dims[2]), device=x.device, dtype=torch.float32)
        arr = _lib.float_array(self._times(time, B))
        with torch.cuda.device(x.device):
            st = torch.cuda.current_stream().cuda_stream
            _lib.check(ctx.L.irsde_trace_forward(ctx.h, ctypes.c_void_p(x.data_ptr()),
                                                 ctypes.c_void_p(cond.data_ptr()) if cond is not None else None, arr, len(arr),
                                                 B, H, W, op, ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(st)), ctx.h)
        return out

    def launch_count(self):
        return int(self._ctx.L.irsde_launch_count(self._ctx.h)) if self._ctx else 0

    def upload_count(self):
        """How many times ``sync_weights`` uploaded the parameters (once per change of their storage or version)."""
        return getattr(self, "_uploads", 0)


class DenoisingUNet(ConditionalUNet):
    """The denoising-sde variant: no condition input, full softmax ``Attention`` at ``mid_attn``
    (codes/config/denoising-sde/models/modules/DenoisingUNet_arch.py:19-133).  The reference class is
    also called ``ConditionalUNet``; ``irsde_b200.denoising_sde.ConditionalUNet`` aliases this one."""

    variant = "denoising"

    def __init__(self, in_nc, out_nc, nf, depth=4, precision=None, force_simt=False):
        super().__init__(in_nc, out_nc, nf, depth, 1, precision, force_simt)

    @torch.no_grad()
    def forward(self, x, time):
        return self._run(x, None, time)


def infer_unet_config(state_dict):
    """(in_nc, out_nc, nf, ch_mult, variant) of a ConditionalUNet state dict in the reference's naming, or None."""
    try:
        sd = state_dict
        nf = sd["init_conv.weight"].shape[0]
        cin0 = sd["init_conv.weight"].shape[1]
        out_nc = sd["final_conv.weight"].shape[0]
        variant = "denoising" if "mid_attn.fn.fn.to_out.weight" in sd else "conditional"
        in_nc = cin0 // 2 if variant == "conditional" else cin0
        mult, i = [], 0
        while ("downs.%d.3.weight" % i) in sd:
            mult.append(sd["downs.%d.3.weight" % i].shape[0] // nf)
            i += 1
        if not mult:
            return None
        return in_nc, out_nc, nf, mult, variant
    except Exception:
        return None

