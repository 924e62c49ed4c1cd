"""Every instantiation of the tap-GEMM conv kernel (conv_tc_persist_kernel<BN, MODE, EKT>) with its fused epilogue, against
an fp64 reference, through irsde_conv2d_fused: the same descriptor, runtime-table and launch calls the launch plan makes,
with the views the plan gives a conv (channel-offset input, output and residual views into wider buffers, a cropped fp32
NCHW head) and the time-modulation table read at a runtime row, shared by the batch or one row per image.  The rows include
the NAFNet downs (2x2/2 over space-to-depth planes) at the BN the selector picks for each width, and the bf16 7x7 stem.

Each case names the <BN, MODE, EKT> it must land on and checks it through the `info` the call returns.  The reference is
the conv of the operands rounded as the engine rounds them (bf16 for engine 1) in fp64, then (acc + bias) * (scale + 1) +
shift (or * mult_vec), SiLU, + residual.  Bounds: bf16 2^-8 |ref| + 1e-3 max|ref| (output rounding and summation order);
fp32x3 max(2e-5 max|ref|, 8x what plain fp32 gets); fp32 SIMT 2e-5.  The SIMT kernel's own matrix is
test_gpu_conv_simt.py; the three SIMT rows here stay for test_fused_conv_refuses_bad_views, which reuses the pitched one.  Before the kernel's output is compared, every
time-modulated case shows that references built from a wrong table row, another image's row, scale and shift exchanged,
or the table shifted by one channel all violate its bound.  Everything outside the conv's output slice (other channels of
the wide buffer, a guard band after the cropped NCHW head) must come back bit-identical.

test_conv_tc_sass.py::test_every_compiled_instantiation_has_a_case runs without a GPU: it fails when the compiled conv_tc.cu
holds an instantiation that no case below names (or a case names one that no longer exists).
"""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

NUM_SMS = 132
QSM, AFF, SILU, RES, GEN = 1, 2, 4, 8, 16  # conv_tc.cu EK_*
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(name, expect, engine, B, Cin, H, W, Cout, K, up=False, bias=False, silu=False, ss=None, t_row=0, mv=False,
          qsm=False, in_view=None, out_view=None, res_view=None, crop=None, min_tiles=0):
    """expect = (BN, MODE, EKT) of the kernel that must run (None: SIMT engine); ss = None | "shared" | "image";
    *_view = (pitch, channel offset) of the wide NHWC buffer (None: dense); crop = (h, w) of the fp32 NCHW head output."""
    return dict(name=name, expect=expect, engine=engine, B=B, Cin=Cin, H=H, W=W, Cout=Cout, K=K, up=up, bias=bias, silu=silu,
                ss=ss, t_row=t_row, mv=mv, qsm=qsm, in_view=in_view or (Cin, 0), out_view=out_view or (Cout, 0),
                res_view=res_view, crop=crop, min_tiles=min_tiles)


CASES = [
    # ---- engine 1 (bf16), per-tap boxes (MODE 0)
    _case("per-tap BN=32: nearest x2 + 3x3, Cin 40 of a 48-ch buffer, Cout 24 into a concat slice, bias, per-image rows",
          (32, 0, GEN), 1, 3, 40, 6, 10, 24, 3, up=True, bias=True, ss="image", t_row=2, in_view=(48, 8), out_view=(40, 8)),
    _case("per-tap BN=64: 4x4/2 downsample, shared row + SiLU + pitched residual", (64, 0, GEN), 1, 2, 32, 16, 24, 64, 4,
          silu=True, ss="shared", t_row=1, res_view=(72, 8)),
    _case("per-tap BN=128: 1x1 Cin 96, bias + residual", (128, 0, GEN), 1, 3, 96, 64, 64, 128, 1, bias=True,
          res_view=(128, 0)),
    _case("per-tap BN=256 block1: 3x3 64->256, per-image rows + SiLU, 288 tiles", (256, 0, GEN), 1, 9, 64, 64, 64, 256, 3,
          silu=True, ss="image", t_row=3, min_tiles=2 * NUM_SMS),
    _case("per-tap BN=64: 1x1 into the upper half of a concat buffer, W < 16", (64, 0, 0), 1, 2, 64, 20, 12, 64, 1,
          out_view=(128, 64)),
    _case("per-tap small problem, BN halved 128 -> 64: 1x1, bias * mult_vec", (64, 0, AFF), 1, 1, 32, 8, 8, 128, 1,
          bias=True, mv=True),
    _case("per-tap BN=128: 1x1 128->128", (128, 0, 0), 1, 3, 128, 64, 64, 128, 1),
    _case("per-tap BN=128 N-fastest: 1x1 192->384 read from a 384-ch buffer (26 MB), bias + shared row", (128, 0, AFF), 1,
          1, 192, 136, 256, 384, 1, bias=True, ss="shared", t_row=2, in_view=(384, 128)),
    _case("per-tap BN=128 to_qkv: 1x1 64->384, q-softmax", (128, 0, QSM), 1, 2, 64, 32, 32, 384, 1, qsm=True),
    _case("per-tap BN=256: 3x3 64->256, ragged 60x50 (BW=8, BH=16), bias + shared row", (256, 0, AFF), 1, 3, 64, 60, 50,
          256, 3, bias=True, ss="shared", t_row=1),
    _case("per-tap BN=256: 1x1 128->512 into a concat slice", (256, 0, 0), 1, 9, 128, 32, 32, 512, 1, out_view=(768, 256)),
    # ---- engine 1 (bf16): the NAFNet downs (2x2/2 over space-to-depth planes, bias) and the 7x7 stem (7 row taps)
    _case("per-tap BN=128: NAFNet downs.0 2x2/2 64->128, bias", (128, 0, AFF), 1, 3, 64, 128, 128, 128, 2, bias=True),
    _case("per-tap BN=256: NAFNet downs.1 2x2/2 128->256, bias", (256, 0, AFF), 1, 2, 128, 256, 256, 256, 2, bias=True),
    _case("per-tap BN halved 256 -> 128: NAFNet downs.2 2x2/2 256->512, bias", (128, 0, AFF), 1, 1, 256, 128, 128, 512, 2,
          bias=True),
    _case("per-tap BN halved 256 -> 64: NAFNet downs.3 2x2/2 512->1024, bias", (64, 0, AFF), 1, 2, 512, 32, 32, 1024, 2,
          bias=True),
    _case("per-tap BN=64 stem: 7x7 Cin 6 in pitch 8 -> 64, into channels 64.. of a 128-ch buffer", (64, 0, 0), 1, 2, 6, 20,
          28, 64, 7, in_view=(8, 0), out_view=(128, 64)),
    _case("per-tap BN=64 stem: 7x7 Cin 3 in pitch 8 -> 64", (64, 0, 0), 1, 2, 3, 32, 24, 64, 7, in_view=(8, 0)),
    _case("per-tap BN=64 stem: 7x7 Cin 6 -> 64, ragged 37x53", (64, 0, 0), 1, 2, 6, 37, 53, 64, 7, in_view=(8, 0)),
    # ---- engine 1 (bf16), ROWS (MODE 2)
    _case("ROWS BN=32: 3x3 24->16, W < 16 (BW=8), H % 16 != 0, bias + SiLU", (32, 2, GEN), 1, 2, 24, 13, 7, 16, 3,
          bias=True, silu=True),
    _case("ROWS BN=32: 3x3 head 64->3, fp32 NCHW cropped to 17x25", (32, 2, GEN), 1, 2, 64, 20, 28, 3, 3, bias=True,
          crop=(17, 25)),
    _case("ROWS BN=64: 3x3 64->64, W % 16 != 0", (64, 2, GEN), 1, 2, 64, 20, 36, 64, 3),
    _case("ROWS BN=128: 3x3 72->128, bias + residual", (128, 2, GEN), 1, 1, 72, 24, 40, 128, 3, bias=True,
          res_view=(128, 0)),
    _case("ROWS BN=64 block1: 3x3 64->64, per-image rows + SiLU, 384 tiles", (64, 2, AFF | SILU), 1, 3, 64, 128, 128, 64, 3,
          silu=True, ss="image", t_row=4, min_tiles=2 * NUM_SMS),
    _case("ROWS BN=64 block2: 3x3 64->64, SiLU + pitched residual, into a concat slice", (64, 2, SILU | RES), 1, 2, 64, 24,
          20, 64, 3, silu=True, res_view=(192, 64), out_view=(128, 64)),
    _case("ROWS BN=128 block1: 3x3 64->128, per-image rows + SiLU, 384 tiles", (128, 2, AFF | SILU), 1, 3, 64, 128, 128,
          128, 3, silu=True, ss="image", t_row=1, min_tiles=2 * NUM_SMS),
    _case("ROWS BN=128 block2 (COMPACT): 3x3 128->128, SiLU + pitched residual, into a concat slice", (128, 2, SILU | RES),
          1, 2, 128, 40, 24, 128, 3, silu=True, res_view=(256, 128), out_view=(256, 0)),
    # ---- engine 2 (fp32x3, MODE 3)
    _case("fp32x3 BN=32: 3x3 head 64->3, fp32 NCHW cropped to 18x25, bias", (32, 3, GEN), 2, 2, 64, 20, 28, 3, 3, bias=True,
          crop=(18, 25)),
    _case("fp32x3 BN=64: 4x4/2 downsample 32->48, bias + per-image rows, into a concat slice", (64, 3, GEN), 2, 3, 32, 16,
          24, 48, 4, bias=True, ss="image", t_row=2, out_view=(64, 12)),
    _case("fp32x3 BN=128 block1: 3x3 64->128, per-image rows + SiLU, 288 tiles", (128, 3, GEN), 2, 9, 64, 64, 64, 128, 3,
          silu=True, ss="image", t_row=3, min_tiles=2 * NUM_SMS),
    _case("fp32x3 BN=128: nearest x2 + 3x3 40->136 (two N tiles), shared row + pitched residual", (128, 3, GEN), 2, 2, 40,
          6, 10, 136, 3, up=True, ss="shared", t_row=5, res_view=(144, 8)),
    _case("fp32x3 BN=128: NAFNet down 2x2/2 64->128, bias", (128, 3, GEN), 2, 3, 64, 128, 128, 128, 2, bias=True),
    # ---- engine 0 (fp32 SIMT)
    _case("SIMT: 3x3 20->12, per-image rows + SiLU + pitched residual, pitched input and output", None, 0, 3, 20, 9, 11, 12,
          3, silu=True, ss="image", t_row=1, in_view=(24, 4), out_view=(20, 8), res_view=(16, 4)),
    _case("SIMT: 3x3 head 16->3, fp32 NCHW cropped to 9x13", None, 0, 2, 16, 10, 14, 3, 3, bias=True, crop=(9, 13)),
    _case("SIMT: nearest x2 + 3x3 8->12, bias * mult_vec", None, 0, 2, 8, 5, 7, 12, 3, up=True, bias=True, mv=True),
]


# ------------------------------------------------------------------------------------------------------------------
# GPU: the instantiation matrix
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


def _geom(c):
    K = c["K"]
    s, p = {4: (2, 1), 2: (2, 0)}.get(K, (1, (K - 1) // 2))  # 4x4/2 pad 1, 2x2/2 pad 0, else KxK/1 "same"
    up = 2 if c["up"] else 1
    return s, p, (c["H"] * up + 2 * p - K) // s + 1, (c["W"] * up + 2 * p - K) // s + 1


def _bf16(t):
    return t.bfloat16().float()


def _data(c, dev):
    """Every buffer of the call, drawn so that a wrong row, image, channel or scale/shift order is visible."""
    g = torch.Generator(device=dev).manual_seed(sum(map(ord, c["name"])))
    B, Cin, H, W, Cout, K = c["B"], c["Cin"], c["H"], c["W"], c["Cout"], c["K"]
    _, _, Ho, Wo = _geom(c)
    rnd = lambda *s: torch.randn(*s, generator=g, device=dev)
    uni = lambda *s: torch.rand(*s, generator=g, device=dev) * 2 - 1
    d = {}
    d["x"] = rnd(B, H, W, c["in_view"][0])  # the whole wide buffer: channels outside the view must not be read
    if c["engine"] == 1:
        d["x"] = _bf16(d["x"])
    d["w"] = rnd(Cout, Cin, K, K) / (Cin * K * K) ** 0.5
    d["bias"] = 0.5 * rnd(Cout) if c["bias"] else None
    d["mv"] = (0.5 + torch.rand(Cout, generator=g, device=dev)) * torch.sign(uni(Cout)) if c["mv"] else None
    if c["ss"]:
        stride = 1 if c["ss"] == "image" else 0
        d["stride"] = stride
        d["rows"] = c["t_row"] + (B - 1) * stride + 2   # room for the row after the last one used
        d["ss_off"] = 16
        d["S"] = d["ss_off"] + 2 * Cout + 8              # room for the table shifted by one channel
        d["ss"] = uni(d["rows"], d["S"])                 # scale + 1 in (0, 2), shift in (-1, 1): O(1) against |acc| ~ 1
    if c["res_view"]:
        d["res"] = _bf16(rnd(B, Ho, Wo, c["res_view"][0]))
    if c["crop"]:
        ch, cw = c["crop"]
        d["y"] = rnd(B * Cout * ch * cw + 4096)          # + guard band
    else:
        d["y"] = _bf16(rnd(B, Ho, Wo, c["out_view"][0]))  # bf16 values: the bf16 engine's round trip keeps them exactly
    return d


def _run(lib, ctx, c, d):
    s, p, Ho, Wo = _geom(c)
    ptr = lambda t: t.data_ptr() if t is not None else None
    ep = lib._lib.ConvEpilogue()
    ep.bias, ep.mult_vec, ep.res = ptr(d["bias"]), ptr(d["mv"]), ptr(d["res"]) if c["res_view"] else None
    ep.silu, ep.flags = int(c["silu"]), 1 if c["qsm"] else 0
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
                                  c["K"], c["K"], s, p, int(c["up"]), info,
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    lib._lib.check(rc, ctx.h)
    torch.cuda.synchronize()
    return y, tuple(info)


def _phase_weights(w, py, px):
    """The bf16 engine's nearest-x2 + 3x3 weights for output phase (py, px): the 3x3 taps that land on one low-res pixel,
    summed in fp32 in the engine's order (engine.cu pack_tc_up_kernel) and then rounded to bf16."""
    sets = {(0, 0): (0,), (0, 1): (1, 2), (1, 0): (0, 1), (1, 1): (2,)}
    out = torch.empty(w.shape[0], w.shape[1], 2, 2, device=w.device)
    for a in range(2):
        for b in range(2):
            acc = torch.zeros_like(w[:, :, 0, 0])
            for r in sets[(py, a)]:
                for q in sets[(px, b)]:
                    acc = acc + w[:, :, r, q]
            out[:, :, a, b] = acc
    return _bf16(out)


def _conv_acc(c, d, dtype):
    """The conv alone, NCHW, in `dtype` on the GPU (fp64: the exact answer for the engine's operands)."""
    s, p, _, _ = _geom(c)
    pitch, off = c["in_view"]
    x = d["x"][..., off:off + c["Cin"]].permute(0, 3, 1, 2).to(dtype)
    w = d["w"]
    if c["engine"] == 1 and c["up"]:
        B, H, W = c["B"], c["H"], c["W"]
        xp = F.pad(x, (1, 1, 1, 1))
        out = torch.empty(B, c["Cout"], 2 * H, 2 * W, device=x.device, dtype=dtype)
        for py in range(2):
            for px in range(2):
                o = F.conv2d(xp, _phase_weights(w, py, px).to(dtype))
                out[:, :, py::2, px::2] = o[:, :, py:py + H, px:px + W]
        return out
    if c["engine"] == 1:
        w = _bf16(w)
    if c["up"]:
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    return F.conv2d(x, w.to(dtype), stride=s, padding=p)


def _epilogue(c, d, acc, rows=None, ss_off=None, swap_ss=False):
    """Reference epilogue in acc's dtype and device.  rows / ss_off / swap_ss override the table lookup (mutations)."""
    y = acc
    B, Cout = c["B"], c["Cout"]
    if c["qsm"]:
        q = y[:, :128].reshape(B, 4, 32, *y.shape[2:]).softmax(dim=2) * 32 ** -0.5
        y = torch.cat([q.reshape(B, 128, *y.shape[2:]), y[:, 128:]], dim=1)
    col = lambda v: v.to(y)[None, :, None, None]
    if d["bias"] is not None:
        y = y + col(d["bias"])
    if c["ss"]:
        if rows is None:
            rows = [c["t_row"] + b * d["stride"] for b in range(B)]
        off = d["ss_off"] if ss_off is None else ss_off
        tab = d["ss"].to(y)[torch.tensor(rows, device=d["ss"].device)]
        scale, shift = tab[:, off:off + Cout], tab[:, off + Cout:off + 2 * Cout]
        if swap_ss:
            scale, shift = shift, scale
        y = y * (scale[:, :, None, None] + 1) + shift[:, :, None, None]
    if d["mv"] is not None:
        y = y * col(d["mv"])
    if c["silu"]:
        y = F.silu(y)
    if c["res_view"]:
        pitch, off = c["res_view"]
        y = y + d["res"][..., off:off + Cout].permute(0, 3, 1, 2).to(y)
    if c["crop"]:
        y = y[:, :, :c["crop"][0], :c["crop"][1]]
    return y


def _mutations(c, d):
    """(label, epilogue overrides) of the wrong-table references the bound must reject."""
    B, t, st = c["B"], c["t_row"], d["stride"]
    rows = [t + b * st for b in range(B)]
    m = [("row t+1", dict(rows=[r + 1 for r in rows])), ("row t-1", dict(rows=[r - 1 for r in rows])),
         ("scale and shift exchanged", dict(swap_ss=True)), ("table shifted by one channel", dict(ss_off=d["ss_off"] + 1))]
    if st:
        m.append(("images 0 and 1 swap rows", dict(rows=[rows[1], rows[0]] + rows[2:])))
    return m


def _over_bound(c, got, ref, err32):
    """Worst error of `got` over the case's bound (<= 1: within it); all fp64 on the CPU."""
    scale = ref.abs().max().item()
    if c["engine"] == 1:
        return ((got - ref).abs() / (2 ** -8 * ref.abs() + 1e-3 * scale)).max().item()
    if c["engine"] == 2:
        return (got - ref).abs().max().item() / max(2e-5 * scale, 8 * err32)
    return (got - ref).abs().max().item() / (2e-5 * max(scale, 1.0))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_fused_conv_vs_fp64(lib, scratch_ctx, case, capsys):
    c = case
    dev = _dev()
    d = _data(c, dev)
    B, Cout = c["B"], c["Cout"]
    acc = _conv_acc(c, d, torch.float64)
    ref = _epilogue(c, d, acc).cpu()
    err32 = 0.0
    if c["engine"] == 2:  # what plain fp32 (cuDNN, TF32 off) gets on the same problem
        err32 = (_epilogue(c, d, _conv_acc(c, d, torch.float32)).double().cpu() - ref).abs().max().item()
    acc_cpu = acc.cpu()
    dcpu = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in d.items()}
    # the bound must reject every wrong-table reference before it is used to accept the kernel
    if c["ss"]:
        for label, kw in _mutations(c, d):
            r = _over_bound(c, _epilogue(c, dcpu, acc_cpu, **kw), ref, err32)
            assert r > 1.0, ("the bound does not see a wrong table lookup", label, r)
    y, info = _run(lib, scratch_ctx, c, d)
    y = y.cpu()
    if c["crop"]:
        n = B * Cout * c["crop"][0] * c["crop"][1]
        got = y[:n].reshape(B, Cout, *c["crop"]).double()
        assert torch.equal(y[n:].view(torch.int32), d["y"][n:].cpu().view(torch.int32)), "write past the cropped output"
    else:
        pitch, off = c["out_view"]
        y0 = d["y"].cpu()
        outside = torch.ones(pitch, dtype=torch.bool)
        outside[off:off + Cout] = False
        assert torch.equal(y[..., outside].view(torch.int32), y0[..., outside].view(torch.int32)), "write outside the slice"
        got = y[..., off:off + Cout].permute(0, 3, 1, 2).double()
    assert got.shape == ref.shape
    r = _over_bound(c, got, ref, err32)
    with capsys.disabled():
        kern = "<%3d,%d,%2d>" % info[:3] if c["expect"] else "SIMT        "
        print("\n  %s tiles %5d  worst err / bound %.3f  %s" % (kern, info[3], r, c["name"]), end="")
    if c["expect"] is not None:
        assert info[:3] == c["expect"], (info, c["expect"])
        assert info[3] >= c["min_tiles"], info
    assert r <= 1.0, (c["name"], r)


@pytest.mark.gpu
def test_fused_conv_refuses_bad_views(lib, scratch_ctx):
    """Host-side validation: each call below describes a view, table row or crop outside what it declares, and must be
    refused.  The SIMT engine uses the caller's buffers directly, and every buffer here has a generous tail, so a check
    that let a call through would still stay inside the allocations."""
    dev = _dev()
    c = CASES[-3]  # SIMT, per-image rows, pitched input / output / residual
    assert c["engine"] == 0 and c["ss"] == "image"
    d = _data(c, dev)
    tail = lambda t: torch.cat([t.reshape(-1), torch.zeros(1 << 16, device=dev)])
    d.update(x=tail(d["x"]), y=tail(d["y"]), res=tail(d["res"]), ss=tail(d["ss"]))
    B, Cout, Cin = c["B"], c["Cout"], c["Cin"]
    _, _, Ho, Wo = _geom(c)
    bad = [dict(t_row=d["rows"] - (B - 1)),                  # the last image's row is past the table
           dict(ss_off=d["S"] - 2 * Cout + 1),                # its shift columns run past the row
           dict(out_view=(20, 12)),                           # 12 + 12 > 20
           dict(out_view=(20, 6)),                            # offset not 16-byte aligned
           dict(in_view=(24, 8)),                             # 8 + 20 > 24
           dict(res_view=(16, 8)),                            # 8 + 12 > 16
           dict(crop=(Ho + 1, Wo), res_view=None),            # crop larger than the output
           dict(mv=True)]                                     # mult_vec together with the time table
    for kw in bad:
        cc = dict(c, **{k: v for k, v in kw.items() if k in c})
        dd = dict(d)
        if "ss_off" in kw:
            dd["ss_off"] = kw["ss_off"]
        if kw.get("mv"):
            dd["mv"] = torch.ones(Cout, device=dev)
        with pytest.raises(lib._lib.IrsdeError):
            _run(lib, scratch_ctx, cc, dd)
    _run(lib, scratch_ctx, c, d)  # the unmodified call is accepted


# ------------------------------------------------------------------------------------------------------------------
# GPU: the runtime time row of the whole network, bit for bit
# ------------------------------------------------------------------------------------------------------------------
def _small_net(lib, precision, dev):
    from oracle import irsde_oracle as O
    P = O.make_weights(3, 3, 16, 3, seed=5)
    net = lib.ConditionalUNet(3, 3, 16, depth=3, precision=precision)
    net.load_state_dict(P, strict=True)
    return net.to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32x3"])
def test_graph_replayed_chain_equals_eager_steps(lib, precision):
    """reverse_sde replays one captured step graph whose convs read the time row through the device step counter (chain
    table); the eager loop runs noise_fn (row 0 of a one-row forward table) + the step kernel: bit-identical."""
    dev = _dev()
    net = _small_net(lib, precision, dev)
    T = 12
    sde = lib.IRSDE(10, T, schedule="cosine", eps=0.005, device=dev)
    sde.use_graph = True
    sde.set_model(net)
    g = torch.Generator().manual_seed(3)
    lq = torch.rand(2, 3, 32, 40, generator=g)
    xT = (lq + torch.randn(lq.shape, generator=g) * sde.max_sigma).to(dev)
    zs = torch.randn((T,) + tuple(lq.shape), generator=g).to(dev)
    sde.set_mu(lq.to(dev))
    a = sde.reverse_sde(xT, zs=zs)
    x = xT.clone()
    for i, t in enumerate(reversed(range(1, T + 1))):
        x = sde._native_step(lib._lib.MODE_SDE, x, sde.mu, sde.noise_fn(x, t), zs[i], t)
    assert torch.equal(a, x), (a - x).abs().max().item()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32x3"])
def test_per_image_time_rows_equal_uniform_batches(lib, precision):
    """A forward with per-image times t_vec: image b equals image b of the same batch run with every image at t_vec[b]
    (same plan and tiles, only the table row differs), bit for bit."""
    dev = _dev()
    net = _small_net(lib, precision, dev)
    g = torch.Generator().manual_seed(6)
    cond = torch.rand(3, 3, 32, 40, generator=g).to(dev)
    x = (cond + torch.randn(3, 3, 32, 40, generator=g).to(dev) * 0.3)
    t_vec = [5, 61, 23]
    y = net(x, cond, torch.tensor(t_vec))
    for b, t in enumerate(t_vec):
        yb = net(x, cond, torch.tensor([t] * 3))
        assert torch.equal(y[b], yb[b]), (b, t, (y[b] - yb[b]).abs().max().item())
    assert not torch.equal(y[0], net(x, cond, torch.tensor([t_vec[1]] * 3))[0])
