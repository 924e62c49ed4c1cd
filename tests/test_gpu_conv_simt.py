"""The SIMT implicit-GEMM conv (conv_simt_kernel) in both storage types against an fp64 reference, through
irsde_conv2d_fused: engine 0 is the fp32 kernel (the fp32 mode's only conv, and the fp32x3 plans' 7x7 stem, NAFNet intro
and latent_conv), engine 3 the bf16 kernel that a bf16 plan gives every conv the tap-GEMM refuses (NAFNet intro, the latent
autoencoder's init_conv / latent_conv / post_latent_conv, every conv of a UNet whose width is not a multiple of 8).

Each case stands for a conv of a plan, with the views the plan gives it, and names the code path it must take: the 4-wide
input gather (vecA), weight load (vecB) and NHWC store (vecO), each on or off, as the call's `info` reports them.  The
reference is the conv in fp64 of the operands as the engine rounds them (bf16 activations and residual on engine 3, fp32
weights on both), then bias -> (scale + 1) * x + shift (or * mult_vec) -> SiLU -> + residual.  Bound:
max(4 * err_cudnn_fp32, 2^-23 * max|ref|), where err_cudnn_fp32 is what cuDNN in fp32 with TF32 off gets on the same
problem; engine 3 adds the bf16 rounding of its NHWC output, 2^-8 |ref|.

Before the kernel's output is compared, every case shows that its bound rejects references built from a conv that drops
the last 16-wide K tile (the partial one where Ktot % 16 != 0), the last 64-pixel M tile or the last 64-channel N tile, or
flips the kernel by 180 degrees; the upsampling case also src = (dst + 1) >> 1, the 2x2/2 case the transposed plane order,
and the time-modulated cases a wrong row, another image's row, scale and shift exchanged and the table shifted by one
channel.  Everything outside the output slice, and a guard band after a cropped NCHW output, must come back bit-identical.

test_plan_simt_convs_have_cases checks that the convs the plan builder sends to this kernel are the ones listed here, and
test_every_compiled_kernel_has_a_case (no GPU) that every kernel of conv_simt.cu, linattn_fused.cu, imaging.cu and
engine.cu is checked by a case here or by a named test elsewhere.
"""
import ast
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

from test_gpu_conv_epilogues import CASES as TC_CASES, _epilogue, _mutations

BM, BN, BK = 64, 64, 16  # conv_simt.cu tile


def _case(name, engine, path, B, Cin, H, W, Cout, K, stride=1, pad=None, up=False, bias=False, silu=False, ss=None, t_row=0,
          mv=False, in_view=None, out_view=None, res_view=None, crop=None):
    """path = (vecA, vecB, vecO) the kernel must take; ss = None | "shared" | "image"; *_view = (pitch, channel offset) of
    the wide NHWC buffer (None: dense); crop = (h, w) of the fp32 NCHW output."""
    return dict(name=name, engine=engine, path=path, B=B, Cin=Cin, H=H, W=W, Cout=Cout, K=K, stride=stride,
                pad=(K - 1) // 2 if pad is None else pad, up=up, bias=bias, silu=silu, ss=ss, t_row=t_row, mv=mv, qsm=False,
                in_view=in_view or (Cin, 0), out_view=out_view or (Cout, 0), res_view=res_view, crop=crop,
                kernels=["conv_simt_kernel<%s>" % ("bf16" if engine == 3 else "float"), "pack_simt_kernel"] +
                (["cast_f32_bf16_kernel", "cast_bf16_f32_kernel"] if engine == 3 else []))


CASES = [
    # ---- engine 3: bf16 storage, the convs a bf16 plan sends to the SIMT kernel
    _case("bf16 NAFNet intro: 3x3 Cin 6 in pitch 8 -> 64, bias, ragged 37x53", 3, (0, 1, 1), 2, 6, 37, 53, 64, 3, bias=True,
          in_view=(8, 0)),
    _case("bf16 denoising-sde NAFNet intro: 3x3 Cin 3 in pitch 8 -> 64, bias", 3, (0, 1, 1), 2, 3, 24, 40, 64, 3, bias=True,
          in_view=(8, 0)),
    _case("bf16 AE init_conv: 3x3 Cin 3 in pitch 8 -> 64", 3, (0, 1, 1), 2, 3, 32, 24, 64, 3, in_view=(8, 0)),
    _case("bf16 AE post_latent_conv: 1x1 Cin 4 in pitch 8 -> 256, into offset 0 of a 512-ch concat buffer", 3, (1, 1, 1), 2, 4,
          12, 20, 256, 1, in_view=(8, 0), out_view=(512, 0)),
    _case("bf16 AE latent_conv: 1x1 256 -> 4, fp32 NCHW", 3, (1, 1, 0), 2, 256, 12, 20, 4, 1, crop=(12, 20)),
    _case("bf16 UNet nf=12 stem: 7x7 Cin 6 in pitch 8 -> 12, into channels 12.. of a 24-ch buffer", 3, (0, 1, 1), 2, 6, 20, 28,
          12, 7, in_view=(8, 0), out_view=(24, 12)),
    _case("bf16 UNet nf=12 resblock: 3x3 12 -> 12 read from a 24-ch buffer, per-image rows + SiLU + pitched residual", 3,
          (1, 1, 1), 3, 12, 20, 28, 12, 3, silu=True, ss="image", t_row=2, in_view=(24, 12), res_view=(24, 12)),
    _case("bf16 UNet nf=12 final_conv: 3x3 12 -> 3, fp32 NCHW cropped to 19x26", 3, (1, 0, 0), 2, 12, 20, 28, 3, 3, bias=True,
          crop=(19, 26)),
    _case("bf16 UNet nf=12 downsample: 4x4/2 12 -> 24, bias", 3, (1, 1, 1), 2, 12, 20, 28, 24, 4, stride=2, pad=1, bias=True),
    _case("bf16 UNet nf=12 upsample: nearest x2 + 3x3 24 -> 12, bias, into channels 0.. of a 36-ch buffer", 3, (1, 1, 1), 2, 24,
          10, 14, 12, 3, up=True, bias=True, out_view=(36, 0)),
    _case("bf16 UNet nf=12 to_qkv: 1x1 12 -> 384", 3, (1, 1, 1), 2, 12, 20, 28, 384, 1),
    _case("bf16 UNet nf=12 to_out: 1x1 128 -> 12, bias", 3, (1, 1, 1), 2, 128, 20, 28, 12, 1, bias=True),
    # ---- engine 0: fp32
    _case("fp32 NAFNet intro: 3x3 Cin 6 in pitch 8 -> 64, bias, ragged 37x53", 0, (0, 1, 1), 2, 6, 37, 53, 64, 3, bias=True,
          in_view=(8, 0)),
    _case("fp32 denoising-sde NAFNet intro: 3x3 Cin 3 in pitch 4 -> 64, bias", 0, (0, 1, 1), 2, 3, 24, 40, 64, 3, bias=True,
          in_view=(4, 0)),
    _case("fp32 AE init_conv: 3x3 Cin 3 in pitch 4 -> 64", 0, (0, 1, 1), 2, 3, 32, 24, 64, 3, in_view=(4, 0)),
    _case("fp32 AE latent_conv: 1x1 256 -> 4, fp32 NCHW", 0, (1, 1, 0), 2, 256, 12, 20, 4, 1, crop=(12, 20)),
    _case("fp32 3x3 512 -> 512 (Ktot 4608), shared row", 0, (1, 1, 1), 1, 512, 16, 16, 512, 3, ss="shared", t_row=1),
    _case("fp32 decoder concat 3x3 1536 -> 512 (Ktot 13824), per-image rows + SiLU", 0, (1, 1, 1), 2, 1536, 8, 8, 512, 3,
          silu=True, ss="image", t_row=3),
    _case("fp32 4x4/2 downsample 64 -> 128, bias", 0, (1, 1, 1), 2, 64, 24, 32, 128, 4, stride=2, pad=1, bias=True),
    _case("fp32 nearest x2 + 3x3 128 -> 64, bias, into a concat slice", 0, (1, 1, 1), 2, 128, 10, 14, 64, 3, up=True,
          bias=True, out_view=(192, 64)),
    _case("fp32 1x1 res_conv 192 -> 64, then the pitched residual", 0, (1, 1, 1), 2, 192, 20, 28, 64, 1, res_view=(128, 64)),
    _case("fp32x3 stem: 7x7 Cin 6 in pitch 8 -> 64, into channels 64.. of a 128-ch buffer", 0, (0, 1, 1), 2, 6, 20, 28, 64, 7,
          in_view=(8, 0), out_view=(128, 64)),
    _case("fp32 NAFNet down: 2x2/2 64 -> 128, bias", 0, (1, 1, 1), 2, 64, 20, 28, 128, 2, stride=2, pad=0, bias=True),
    _case("fp32 3x3 head 64 -> 3, fp32 NCHW cropped to 19x26, bias", 0, (1, 0, 0), 2, 64, 20, 28, 3, 3, bias=True,
          crop=(19, 26)),
    _case("fp32 3x3 72 -> 136 (three N tiles, the last partial; Ktot 648)", 0, (1, 1, 1), 2, 72, 9, 11, 136, 3),
    _case("fp32 3x3 Cin 10 in pitch 12 -> 6, NHWC pitch 8", 0, (0, 0, 1), 2, 10, 13, 9, 6, 3, bias=True, in_view=(12, 0),
          out_view=(8, 0)),
    _case("fp32 3x3 Cin 10 in pitch 12 -> 6, fp32 NCHW", 0, (0, 0, 0), 2, 10, 13, 9, 6, 3, bias=True, in_view=(12, 0),
          crop=(13, 9)),
    _case("fp32 1x1 64 -> 64, bias * mult_vec", 0, (1, 1, 1), 2, 64, 20, 28, 64, 1, bias=True, mv=True),
    _case("fp32 one 2048x2048 level: 1x1 64 -> 64, bias", 0, (1, 1, 1), 1, 64, 2048, 2048, 64, 1, bias=True),
]


def _named(prefix):
    """The name of the one case whose name starts with `prefix`."""
    found = [c["name"] for c in CASES if c["name"].startswith(prefix)]
    assert len(found) == 1, (prefix, found)
    return found[0]


# Every conv a launch plan sends to the SIMT kernel (bf16 plans: engine 3, fp32x3 plans: engine 0), by weight name, with
# the case that stands for it.  test_plan_simt_convs_have_cases fails when a plan routes a conv that is not listed.
_NAF_INTRO = {"intro.weight": "bf16 NAFNet intro"}
_DSDE_INTRO = {"intro.weight": "bf16 denoising-sde NAFNet intro"}
_AE = {"init_conv.weight": "bf16 AE init_conv", "latent_conv.weight": "bf16 AE latent_conv"}
_UNET12_RES = "bf16 UNet nf=12 resblock"
PLAN_SIMT = {
    ("bf16", "ConditionalNAFNet"): _NAF_INTRO,
    ("bf16", "ConditionalNAFNet latent"): {},
    ("bf16", "DenoisingNAFNet"): _DSDE_INTRO,
    ("bf16", "latent UNet"): _AE,
    ("bf16", "ConditionalUNet nf=64"): {},
    ("bf16", "ConditionalUNet nf=12"): dict(
        {"init_conv.weight": "bf16 UNet nf=12 stem", "final_conv.weight": "bf16 UNet nf=12 final_conv",
         "downs.0.3.weight": "bf16 UNet nf=12 downsample", "ups.2.3.1.weight": "bf16 UNet nf=12 upsample",
         "downs.0.2.fn.fn.to_qkv.weight": "bf16 UNet nf=12 to_qkv", "downs.0.2.fn.fn.to_out.0.weight": "bf16 UNet nf=12 to_out"},
        **{n: _UNET12_RES for n in ("downs.0.0.block1.proj.weight", "downs.0.0.block2.proj.weight",
                                    "downs.0.1.block1.proj.weight", "downs.0.1.block2.proj.weight",
                                    "ups.3.0.block1.proj.weight", "ups.3.0.block2.proj.weight", "ups.3.0.res_conv.weight",
                                    "ups.3.1.block1.proj.weight", "ups.3.1.res_conv.weight", "ups.3.3.weight",
                                    "final_res_block.block1.proj.weight", "final_res_block.block2.proj.weight",
                                    "final_res_block.res_conv.weight")}),
    ("fp32x3", "ConditionalNAFNet"): {"intro.weight": "fp32 NAFNet intro"},
    ("fp32x3", "ConditionalNAFNet latent"): {},
    ("fp32x3", "DenoisingNAFNet"): {"intro.weight": "fp32 denoising-sde NAFNet intro"},
    ("fp32x3", "latent UNet"): {"init_conv.weight": "fp32 AE init_conv", "latent_conv.weight": "fp32 AE latent_conv"},
}


# ------------------------------------------------------------------------------------------------------------------
# GPU: the SIMT matrix
# ------------------------------------------------------------------------------------------------------------------
def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lib():
    import irsde_b200
    return irsde_b200


@pytest.fixture(scope="module")
def scratch_ctx(lib):
    _dev()
    return lib._lib.Context(3, 3, 8, 2, lib._lib.NET_CONDITIONAL, lib._lib.PREC_FP32, 0)


def _out_hw(c):
    up = 2 if c["up"] else 1
    return ((c["H"] * up + 2 * c["pad"] - c["K"]) // c["stride"] + 1, (c["W"] * up + 2 * c["pad"] - c["K"]) // c["stride"] + 1)


def _bf16(t):
    return t.bfloat16().float()


def _data(c, dev):
    g = torch.Generator(device=dev).manual_seed(sum(map(ord, c["name"])))
    B, Cin, Cout, K = c["B"], c["Cin"], c["Cout"], c["K"]
    Ho, Wo = _out_hw(c)
    rnd = lambda *s: torch.randn(*s, generator=g, device=dev)
    uni = lambda *s: torch.rand(*s, generator=g, device=dev) * 2 - 1
    rd = _bf16 if c["engine"] == 3 else (lambda t: t)  # engine 3 stages x, res and y in bf16: bf16 values pass unchanged
    d = {"x": rd(rnd(B, c["H"], c["W"], c["in_view"][0])), "w": rnd(Cout, Cin, K, K) / (Cin * K * K) ** 0.5}
    d["bias"] = 0.5 * rnd(Cout) if c["bias"] else None
    d["mv"] = (0.5 + torch.rand(Cout, generator=g, device=dev)) * torch.sign(uni(Cout)) if c["mv"] else None
    if c["ss"]:
        d["stride"] = 1 if c["ss"] == "image" else 0
        d["rows"] = c["t_row"] + (B - 1) * d["stride"] + 2
        d["ss_off"] = 16
        d["S"] = d["ss_off"] + 2 * Cout + 8
        d["ss"] = uni(d["rows"], d["S"])
    if c["res_view"]:
        d["res"] = rd(rnd(B, Ho, Wo, c["res_view"][0]))
    if c["crop"]:
        d["y"] = rnd(B * Cout * c["crop"][0] * c["crop"][1] + 4096)  # + guard band
    else:
        d["y"] = rd(rnd(B, Ho, Wo, c["out_view"][0]))
    return d


def _run(lib, ctx, c, d):
    ptr = lambda t: t.data_ptr() if t is not None else None
    ep = lib._lib.ConvEpilogue()
    ep.bias, ep.mult_vec, ep.res = ptr(d["bias"]), ptr(d["mv"]), ptr(d["res"]) if c["res_view"] else None
    ep.silu = int(c["silu"])
    if c["ss"]:
        ep.ss, ep.ss_rows, ep.ss_S, ep.ss_off = ptr(d["ss"]), d["rows"], d["S"], d["ss_off"]
        ep.ss_img_stride, ep.t_row = d["stride"], c["t_row"]
    if c["res_view"]:
        ep.res_pitch, ep.res_off = c["res_view"]
    ep.in_pitch, ep.in_off = c["in_view"]
    ep.out_pitch, ep.out_off = c["out_view"]
    if c["crop"]:
        ep.crop_h, ep.crop_w = c["crop"]
    y = d["y"].clone()
    info = (ctypes.c_int32 * 4)()
    rc = ctx.L.irsde_conv2d_fused(ctx.h, c["engine"], ctypes.c_void_p(d["x"].data_ptr()), ctypes.c_void_p(d["w"].data_ptr()),
                                  ctypes.byref(ep), ctypes.c_void_p(y.data_ptr()), c["B"], c["Cin"], c["H"], c["W"], c["Cout"],
                                  c["K"], c["K"], c["stride"], c["pad"], int(c["up"]), info,
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    lib._lib.check(rc, ctx.h)
    torch.cuda.synchronize()
    return y, tuple(info)


def _conv_acc(c, d, dtype, w=None, upsample=None):
    """The conv alone, NCHW, in `dtype` (fp64: exact for the engine's operands).  w / upsample override the weights and the
    nearest-x2 gather (mutations)."""
    off = c["in_view"][1]
    x = d["x"][..., off:off + c["Cin"]].permute(0, 3, 1, 2).to(dtype)
    if c["up"]:
        x = upsample(x) if upsample else F.interpolate(x, scale_factor=2, mode="nearest")
    return F.conv2d(x, (d["w"] if w is None else w).to(dtype), stride=c["stride"], padding=c["pad"])


def _src_plus_one(x):
    """Nearest x2 with src = (dst + 1) >> 1 (clamped at the last row / column) instead of dst >> 1."""
    H, W = x.shape[2], x.shape[3]
    ih = ((torch.arange(2 * H, device=x.device) + 1) >> 1).clamp(max=H - 1)
    iw = ((torch.arange(2 * W, device=x.device) + 1) >> 1).clamp(max=W - 1)
    return x[:, :, ih][:, :, :, iw]


def _conv_mutations(c, d):
    """(label, fp64 acc) of the wrong convolutions the bound must reject."""
    B, Cin, Cout, K = c["B"], c["Cin"], c["Cout"], c["K"]
    acc = lambda **kw: _conv_acc(c, d, torch.float64, **kw)
    out = []
    # K index k = (r * K + s) * Cin + ci (the packed [KH*KW][Cin][Cout] rows); drop the last 16-wide tile
    Ktot = K * K * Cin
    k0 = (Ktot - 1) // BK * BK
    kk = torch.arange(Ktot, device=d["w"].device)
    keep = (kk < k0).to(d["w"].dtype).reshape(K, K, Cin).permute(2, 0, 1)
    out.append(("last %s K tile dropped (k >= %d of %d)" % ("partial" if Ktot % BK else "16-wide", k0, Ktot),
                acc(w=d["w"] * keep[None])))
    full = acc()
    Ho, Wo = _out_hw(c)
    M = B * Ho * Wo
    m = full.permute(0, 2, 3, 1).reshape(M, Cout).clone()
    m[(M - 1) // BM * BM:] = 0
    out.append(("last M tile dropped", m.reshape(B, Ho, Wo, Cout).permute(0, 3, 1, 2)))
    n = full.clone()
    n[:, (Cout - 1) // BN * BN:] = 0
    out.append(("last N tile dropped", n))
    if K > 1:
        out.append(("kernel flipped by 180 degrees", acc(w=d["w"].flip(2, 3))))
    if c["up"]:
        out.append(("src = (dst + 1) >> 1", acc(upsample=_src_plus_one)))
    if K == 2 and c["stride"] == 2:
        out.append(("plane order transposed", acc(w=d["w"].transpose(2, 3))))
    return out


def _ratio(c, got, ref, err32):
    """Worst error of `got` over the case's bound (<= 1: within it), on the GPU in fp64."""
    floor = max(4 * err32, 2.0 ** -23 * ref.abs().max().item())
    if c["engine"] == 3 and not c["crop"]:  # the bf16 output's rounding (the NCHW output is fp32)
        return ((got - ref).abs() / (2.0 ** -8 * ref.abs() + floor)).max().item()
    return (got - ref).abs().max().item() / floor


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_simt_conv_vs_fp64(lib, scratch_ctx, case, capsys):
    c = case
    dev = _dev()
    d = _data(c, dev)
    B, Cout = c["B"], c["Cout"]
    ref = _epilogue(c, d, _conv_acc(c, d, torch.float64))
    err32 = (_epilogue(c, d, _conv_acc(c, d, torch.float32)).double() - ref).abs().max().item()
    # the bound must reject every wrong reference before it is used to accept the kernel
    worst_mut = float("inf")
    for label, acc in _conv_mutations(c, d):
        r = _ratio(c, _epilogue(c, d, acc), ref, err32)
        assert r > 1.0, ("the bound does not see a wrong conv", label, r)
        worst_mut = min(worst_mut, r)
    if c["ss"]:
        full = _conv_acc(c, d, torch.float64)
        for label, kw in _mutations(c, d):
            r = _ratio(c, _epilogue(c, d, full, **kw), ref, err32)
            assert r > 1.0, ("the bound does not see a wrong table lookup", label, r)
            worst_mut = min(worst_mut, r)
    y, info = _run(lib, scratch_ctx, c, d)
    y0 = d["y"]
    if c["crop"]:
        n = B * Cout * c["crop"][0] * c["crop"][1]
        got = y[:n].reshape(B, Cout, *c["crop"]).double()
        assert torch.equal(y[n:].view(torch.int32), y0[n:].view(torch.int32)), "write past the cropped output"
    else:
        pitch, off = c["out_view"]
        outside = torch.ones(pitch, dtype=torch.bool, device=dev)
        outside[off:off + Cout] = False
        assert torch.equal(y[..., outside].view(torch.int32), y0[..., outside].view(torch.int32)), "write outside the slice"
        got = y[..., off:off + Cout].permute(0, 3, 1, 2).double()
    assert got.shape == ref.shape
    r = _ratio(c, got, ref, err32)
    with capsys.disabled():
        print("\n  vecA/vecB/vecO %d/%d/%d blocks %6d  worst err / bound %.3f  (mutations >= %.3g)  %s"
              % (info + (r, worst_mut, c["name"])), end="")
    assert info[:3] == c["path"], (info, c["path"])
    assert r <= 1.0, (c["name"], r)


def test_simt_engines_reach_every_path():
    """Each of vecA, vecB and vecO is taken on and off by cases of both storage types."""
    for engine in (0, 3):
        for i in range(3):
            assert {c["path"][i] for c in CASES if c["engine"] == engine} == {0, 1}, (engine, i)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the plans' SIMT convs are the ones the matrix covers
# ------------------------------------------------------------------------------------------------------------------
def _plan_net(lib, precision, kind):
    if kind == "ConditionalNAFNet":
        return lib.ConditionalNAFNet(3, 64, 1, [1, 1, 1, 1], [1, 1, 1, 1], precision=precision)
    if kind == "ConditionalNAFNet latent":
        return lib.ConditionalNAFNet(4, 64, 1, [1, 1, 1, 2], [1, 1, 1, 1], latent=True, precision=precision)
    if kind == "DenoisingNAFNet":
        return lib.DenoisingNAFNet(3, 64, 1, [1, 1, 1, 1], [1, 1, 1, 1], precision=precision)
    if kind == "latent UNet":
        return lib.UNet(3, 3, 64, [1, 2, 4], 4, precision=precision)
    nf = int(kind.split("=")[1])
    return lib.ConditionalUNet(3, 3, nf, depth=4, precision=precision)


@pytest.mark.gpu
def test_plan_simt_convs_have_cases(lib):
    """Walks the launch plan of each network (irsde_plan_op_info; category 1 = CAT_SIMT) and compares the weights it runs on
    the SIMT kernel with PLAN_SIMT, each of which names a case above.  A plan that starts routing a new conv to the SIMT
    kernel fails here until a case covers it.  (irsde_plan_op_info lists the latent autoencoder's encode half.)"""
    dev = _dev()
    CAT_SIMT = 1
    for layers in PLAN_SIMT.values():
        for prefix in layers.values():
            _named(prefix)
    bad = {}
    for (precision, kind), want in PLAN_SIMT.items():
        net = _plan_net(lib, precision, kind).to(dev)
        H = W = 32 if "latent" in kind else 64
        got = {label.split()[0] for label, _, cat in net.plan_ops(1, H, W, dev) if cat == CAT_SIMT}
        if got != set(want):
            bad[(precision, kind)] = ("routed to SIMT", sorted(got), "listed", sorted(want))
        del net
    assert not bad, "\n".join("%s: %s" % kv for kv in bad.items())


# ------------------------------------------------------------------------------------------------------------------
# (CPU) every kernel of conv_simt.cu, linattn_fused.cu, imaging.cu and engine.cu has a case
# ------------------------------------------------------------------------------------------------------------------
# kernels the cases here do not reach, and the test function that checks each
COVERED_ELSEWHERE = {
    "la_kv_ln_kernel<64>": ("test_gpu_linattn_fused.py", "test_linattn_block_vs_fp64"),
    "la_kv_ln_kernel<128>": ("test_gpu_linattn_fused.py", "test_linattn_block_vs_fp64"),
    "la_out_ln_kernel<64>": ("test_gpu_linattn_fused.py", "test_linattn_block_vs_fp64"),
    "la_out_ln_kernel<128>": ("test_gpu_linattn_fused.py", "test_linattn_block_vs_fp64"),
    "tensor2img_kernel": ("test_gpu_parity.py", "test_imaging_bit_exact_vs_reference"),
    "img2tensor_kernel": ("test_gpu_parity.py", "test_imaging_bit_exact_vs_reference"),
    "sqerr_u8_kernel": ("test_gpu_parity.py", "test_imaging_batched_vs_oracle"),
    "ssim_kernel": ("test_gpu_parity.py", "test_imaging_batched_vs_oracle"),
    "ssim_reduce_kernel": ("test_gpu_parity.py", "test_imaging_batched_vs_oracle"),
}


def _tc_case_kernels():
    """The engine.cu kernels that test_gpu_conv_epilogues.CASES reach: weight packers and the bf16 staging casts."""
    k = set()
    for c in TC_CASES:
        if c["engine"] == 0:
            continue
        T = "bf16" if c["engine"] == 1 else "float"
        if c["K"] == 7:
            k.add("pack_tc_stem_kernel")
        elif c["up"]:
            k.add("pack_tc_up_kernel<%s>" % T)
        else:
            k.add("pack_tc_taps_kernel<%s>" % T)
        if c["engine"] == 1:
            k |= {"cast_f32_bf16_kernel", "cast_bf16_f32_kernel"}
    return k


def _normalize(demangled):
    m = re.search(r"(\w+(?:<[^>]*>)?)\(", demangled)
    return m.group(1).replace("(int)", "").replace(" ", "").replace("__nv_bfloat16", "bf16")


def test_every_compiled_kernel_has_a_case(tmp_path):
    here = os.path.dirname(os.path.abspath(__file__))
    for fname, func in set(COVERED_ELSEWHERE.values()):  # the table names tests that exist
        tree = ast.parse(open(os.path.join(here, fname)).read())
        assert func in {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}, (fname, func)
    from test_conv_tc_sass import _build_module
    b = _build_module()
    nvcc = b.NVCC if os.path.isfile(b.NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    tools = os.path.dirname(nvcc)
    cuobjdump, cufilt = os.path.join(tools, "cuobjdump"), os.path.join(tools, "cu++filt")
    if not (os.path.isfile(cuobjdump) and os.path.isfile(cufilt)):
        pytest.skip("cuobjdump / cu++filt not available")
    srcs = ("conv_simt.cu", "linattn_fused.cu", "imaging.cu", "engine.cu")
    procs = {src: subprocess.Popen([nvcc] + b.FLAGS + ["-c", os.path.join(b.CSRC, src), "-o", str(tmp_path / (src + ".o"))],
                                   stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for src in srcs}
    compiled = {}
    for src, p in procs.items():
        out, _ = p.communicate()
        assert p.returncode == 0, out
        s = subprocess.run([cuobjdump, "-res-usage", str(tmp_path / (src + ".o"))], capture_output=True, text=True, check=True)
        mangled = re.findall(r"Function (\S+?):", s.stdout)
        dem = subprocess.run([cufilt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.split("\n")
        compiled[src] = {_normalize(x) for x in dem if x.strip()}
    counts = {src: len(k) for src, k in compiled.items()}
    assert counts == {"conv_simt.cu": 2, "linattn_fused.cu": 4, "imaging.cu": 5, "engine.cu": 8}, compiled
    named = {k for c in CASES for k in c["kernels"]} | _tc_case_kernels() | set(COVERED_ELSEWHERE)
    allk = set().union(*compiled.values())
    assert allk == named, ("without a case", sorted(allk - named), "not compiled", sorted(named - allk))
