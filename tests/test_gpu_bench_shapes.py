"""The BENCHMARKED kernels at BENCHMARK shapes against an independent reference (round-1 verdict, weak #1).

`conv_tc_persist_kernel` runs min(tiles, 132) persistent CTAs (one per H100 SM); every case below has >= 2 x 132 output tiles
per launch, so the multi-tile loop, the producer running ahead into the next tile and the mbarrier phase wrap are compared with an implementation that
shares nothing with them: torch's fp32 convolution (TF32 off) on the bf16-rounded operands, on the same GPU.  The only
differences left are the fp32 summation order and the final rounding of the output to bf16, hence
|y - ref| <= 2^-8 |ref| + 1e-3 * max|ref| elementwise.

Then one full nf=64 / depth=4 forward at 2x3x256x256 (BASELINE config 2's network and image size) in bf16 against the
CPU oracle, with a per-layer error report read back through irsde_trace_forward, the bf16 denoising-sde network, NAFNet
at width 64, and the drift of a T=100 bf16 chain against the fp32 parity mode.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import irsde_oracle as O

NUM_SMS = 132


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


def _conv_ex(lib, ctx, x, w, bias, res, stride, pad, up, silu, flags):
    B, Cin, H, W = x.shape
    if flags & 2:
        Cout, KH, KW = w.shape[1], 1, 1
    else:
        Cout, _, KH, KW = w.shape
    Ho = (H * (2 if up else 1) + 2 * pad - KH) // stride + 1
    Wo = (W * (2 if up else 1) + 2 * pad - KW) // stride + 1
    y = torch.empty(B, Cout, Ho, Wo, device=x.device)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    rc = ctx.L.irsde_conv2d_ex(ctx.h, 1, p(x.contiguous()), p(w.contiguous()), p(bias), p(res), p(y), B, Cin, H, W, Cout, KH, KW,
                               stride, pad, 1 if up else 0, 1 if silu else 0, flags,
                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    lib._lib.check(rc, ctx.h)
    torch.cuda.synchronize()
    return y


def _tiles(B, H, W, Cout, up=False, stride=1):
    """Output tiles of one launch: 128-pixel M tiles x BN-wide N tiles (conv_tc.cu tc_conv_create)."""
    Ha, Wa = (H // stride, W // stride)
    m = B * math.ceil(Ha * Wa / 128) * (4 if up else 1)
    BN = 256 if Cout >= 256 else (128 if Cout > 64 else (64 if Cout > 32 else 32))
    if BN == 256 and Cout % 256 and Cout % 128 == 0:
        BN = 128
    return m * math.ceil(Cout / BN)


BENCH_CONVS = [
    # name, B, Cin, H, W, Cout, K, stride, pad, up, bias, silu, residual
    ("ups.0 block1 3x3 1536->1024 @32^2 (BN=256, K=13824)", 10, 1536, 32, 32, 1024, 3, 1, 1, False, False, True, False),
    ("downs.0 block 3x3 64->64 @256^2 (ROWS, BN=64)", 1, 64, 256, 256, 64, 3, 1, 1, False, False, True, True),
    ("ups.3 block1 3x3 192->128 @256^2 (ROWS, BN=128)", 1, 192, 256, 256, 128, 3, 1, 1, False, False, True, False),
    ("ups.3 res_conv 1x1 192->128 @256^2", 1, 192, 256, 256, 128, 1, 1, 0, False, False, False, False),
    ("downs.0 Downsample 4x4 s2 64->128 @256^2", 3, 64, 256, 256, 128, 4, 2, 1, False, True, False, False),
    ("ups.2 Upsample nearest x2 + 3x3 256->128 @128^2->256^2", 1, 256, 128, 128, 128, 3, 1, 1, True, True, False, False),
    ("mid 3x3 1024->1024 @32^2 (BN=256)", 10, 1024, 32, 32, 1024, 3, 1, 1, False, False, True, True),
    ("ups.1 block1 3x3 768->512 @64^2 (BN=256)", 5, 768, 64, 64, 512, 3, 1, 1, False, False, True, False),
    ("stem 7x7 6->64 @256^2", 2, 6, 256, 256, 64, 7, 1, 3, False, False, False, False),
    ("head 3x3 64->3 @256^2 fp32 NCHW epilogue", 4, 64, 256, 256, 3, 3, 1, 1, False, True, False, False),
]


@pytest.mark.parametrize("case", BENCH_CONVS, ids=[c[0] for c in BENCH_CONVS])
def test_conv_tcgen05_multi_tile_vs_torch(lib, scratch_ctx, case):
    name, B, Cin, H, W, Cout, K, s, p, up, hb, silu, has_res = case
    dev = _dev()
    assert _tiles(B, H, W, Cout, up, s) >= 2 * NUM_SMS, "case must give every persistent CTA at least 2 tiles"
    g = torch.Generator(device=dev).manual_seed(len(name) + Cin + Cout)
    x = torch.randn(B, Cin, H, W, generator=g, device=dev).bfloat16().float()
    w = torch.randn(Cout, Cin, K, K, generator=g, device=dev) / (Cin * K * K) ** 0.5
    b = torch.randn(Cout, generator=g, device=dev) if hb else None
    Ho = (H * (2 if up else 1) + 2 * p - K) // s + 1
    Wo = (W * (2 if up else 1) + 2 * p - K) // s + 1
    res = torch.randn(B, Cout, Ho, Wo, generator=g, device=dev).bfloat16().float() if has_res else None
    y = _conv_ex(lib, scratch_ctx, x, w, b, res, s, p, up, silu, 0)
    xin = F.interpolate(x, scale_factor=2, mode="nearest") if up else x
    # nearest x2 + 3x3: the engine pre-sums the 3x3 taps that fall on one low-res pixel (fp32) BEFORE rounding to bf16, so
    # its weights are not the bf16 rounding of w; compare with the fp32 weights and a tolerance of one bf16 weight ulp
    wref = w if up else w.bfloat16().float()
    ref = F.conv2d(xin, wref, b, stride=s, padding=p)
    if silu:
        ref = F.silu(ref)
    if res is not None:
        ref = ref + res
    scale = ref.abs().max().item()
    rtol, atol = (2 ** -8, 1e-3 * scale) if not up else (2 ** -7, 8e-3 * scale)
    err = (y - ref).abs() - rtol * ref.abs()
    assert err.max().item() <= atol, (name, err.max().item(), scale)


@pytest.mark.parametrize("B,Cin,H,W", [(16, 1024, 32, 32), (1, 128, 256, 256), (2, 64, 256, 256), (3, 128, 128, 128)],
                         ids=["32^2 C=1024", "256^2 C=128 (N-fastest tile order)", "256^2 C=64 (N-fastest)", "128^2 C=128"])
def test_to_qkv_qsoftmax_epilogue_vs_torch(lib, scratch_ctx, B, Cin, H, W):
    """LinearAttention's to_qkv: 1x1 C->384 whose epilogue applies softmax_d(q) * 32^-0.5 per head (module_util.py:165-171)
    to output channels < 128 - at the 32^2 level and at the 256^2 / 128^2 levels, where the input is larger than L2 and the
    three N tiles of one pixel tile are processed back to back (N-fastest tile order, conv_tc.cu tc_conv_create)."""
    dev = _dev()
    assert _tiles(B, H, W, 384) >= 2 * NUM_SMS
    g = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(B, Cin, H, W, generator=g, device=dev).bfloat16().float()
    w = torch.randn(384, Cin, 1, 1, generator=g, device=dev) / Cin ** 0.5 * 3.0   # logits of a few units
    y = _conv_ex(lib, scratch_ctx, x, w, None, None, 1, 0, False, False, 1)
    ref = F.conv2d(x, w.bfloat16().float())
    q = ref[:, :128].reshape(B, 4, 32, H, W).softmax(dim=2) * 32 ** -0.5
    ref = torch.cat([q.reshape(B, 128, H, W), ref[:, 128:]], dim=1)
    scale = ref.abs().max().item()
    err = (y - ref).abs() - 2 ** -8 * ref.abs()
    assert err.max().item() <= 1e-3 * scale, (err.max().item(), scale)
    assert (y[:, :128].reshape(B, 4, 32, H, W).sum(2) - 32 ** -0.5).abs().max().item() < 2e-2  # each head sums to 32^-.5 (bf16 terms)


@pytest.mark.parametrize("B,H,W,Cout", [(2, 256, 256, 64), (3, 256, 256, 128), (5, 128, 128, 256)],
                         ids=["256^2 Cout=64", "256^2 Cout=128, 3 images", "128^2 Cout=256"])
def test_to_out_per_image_weights_vs_torch(lib, scratch_ctx, B, H, W, Cout):
    """The re-associated second einsum + to_out of LinearAttention (module_util.py:176-178): ONE 1x1 GEMM whose [Cout,128]
    matrix differs per image (third TMA coordinate of the weight tensor = image index)."""
    dev = _dev()
    Cin = 128
    assert _tiles(B, H, W, Cout) >= 2 * NUM_SMS
    g = torch.Generator(device=dev).manual_seed(11)
    x = torch.randn(B, Cin, H, W, generator=g, device=dev).bfloat16().float()
    w = torch.randn(B, Cout, Cin, generator=g, device=dev) / Cin ** 0.5
    b = torch.randn(Cout, generator=g, device=dev)
    y = _conv_ex(lib, scratch_ctx, x, w, b, None, 1, 0, False, False, 2)
    ref = torch.einsum("boc,bchw->bohw", w.bfloat16().float(), x) + b[None, :, None, None]
    scale = ref.abs().max().item()
    err = (y - ref).abs() - 2 ** -8 * ref.abs()
    assert err.max().item() <= 1e-3 * scale, (err.max().item(), scale)
    assert not torch.allclose(y[0], (torch.einsum("oc,chw->ohw", w[1].bfloat16().float(), x[0]) + b[:, None, None]), atol=0.1)
    assert torch.isfinite(y).all()


# ------------------------------------------------------------------------------------------------------------------
# full network at the benchmark architecture and image size
# ------------------------------------------------------------------------------------------------------------------
def _layer_report(net, P, xt, cond, t, nf, depth, variant="conditional"):
    """[(label, max|d|, max|ref|, rel_rms)] for every op of the launch plan whose output the oracle checkpoints."""
    tr = {}
    yo = O.unet_forward(P, xt, cond, t, nf, depth, variant=variant, trace=tr)
    dev = _dev()
    B, _, H, W = xt.shape
    rows = []
    xg, cg = xt.to(dev), (cond.to(dev) if cond is not None else None)
    for i, (label, dims, cat) in enumerate(net.plan_ops(B, H, W, dev)):
        if dims is None:
            continue
        key = label if label in tr else label.split(" ")[0]
        if key not in tr or "to_qkv" in key:
            continue
        ref = tr[key]
        got = net.trace(xg, cg, t, i).cpu()
        assert got.shape == ref.shape, (label, got.shape, ref.shape)
        d = (got - ref)
        rows.append((key, d.abs().max().item(), ref.abs().max().item(), (d.pow(2).mean() / ref.pow(2).mean()).sqrt().item()))
    return yo, rows


def test_unet_nf64_forward_bf16_vs_oracle_per_layer(lib, capsys):
    """ConditionalUNet(nf=64, depth=4) on 2x3x256x256 - every layer shape of BASELINE config 2, >= 132 tiles on every
    256^2/128^2 launch - bf16 tensor-core path vs the fp32 CPU oracle: each checkpointed layer within 1.5 % relative RMS and
    3 % of the layer's max (a bf16 pipeline: 2^-9 per rounding, ~60 roundings deep; measured 0.2-0.95 % rel-rms growing
    with depth), output within 4 % of its scale (measured 2.1 %)."""
    dev = _dev()
    nf, depth = 64, 4
    P = O.make_weights(3, 3, nf, depth, seed=0)
    net = lib.ConditionalUNet(3, 3, nf, depth=depth, precision="bf16")
    net.load_state_dict(P, strict=True)
    net = net.to(dev)
    g = torch.Generator().manual_seed(1234)
    cond = torch.rand(2, 3, 256, 256, generator=g)
    xt = cond + torch.randn(2, 3, 256, 256, generator=g) * (10 / 255)
    t = 57
    yo, rows = _layer_report(net, P, xt, cond, t, nf, depth)
    y = net(xt.to(dev), cond.to(dev), t).cpu()
    with capsys.disabled():
        print("\nper-layer bf16 (tensor cores) vs fp32 oracle, nf=64 depth=4, 2x3x256x256, t=%d" % t)
        for key, dmax, rmax, rel in rows:
            print("  %-38s max|d| %.3e  max|ref| %.3e  rel-rms %.2e" % (key, dmax, rmax, rel))
        print("  %-38s max|d| %.3e  max|ref| %.3e" % ("output (eps-hat)", (y - yo).abs().max().item(), yo.abs().max().item()))
    assert len(rows) >= 60
    for key, dmax, rmax, rel in rows:
        assert rel < 1.5e-2 and dmax < 3e-2 * rmax, (key, dmax, rmax, rel)
    assert (y - yo).abs().max().item() < 4e-2 * yo.abs().max().item()


def test_unet_nf64_forward_fp32_vs_oracle(lib):
    """Same network and size in the fp32 parity mode: 1e-4 per forward."""
    dev = _dev()
    nf, depth = 64, 4
    P = O.make_weights(3, 3, nf, depth, seed=0)
    net = lib.ConditionalUNet(3, 3, nf, depth=depth, precision="fp32")
    net.load_state_dict(P, strict=True)
    net = net.to(dev)
    g = torch.Generator().manual_seed(1234)
    cond = torch.rand(1, 3, 256, 256, generator=g)
    xt = cond + torch.randn(1, 3, 256, 256, generator=g) * (10 / 255)
    yo = O.unet_forward(P, xt, cond, 57, nf, depth)
    y = net(xt.to(dev), cond.to(dev), 57).cpu()
    assert (y - yo).abs().max().item() < 1e-4, (y - yo).abs().max().item()


@pytest.mark.parametrize("nf,depth,H,W", [(32, 3, 128, 128), (16, 2, 50, 38), (16, 2, 256, 256)],
                         ids=["N=1024 keys", "ragged N=520 keys", "N=4096 keys"])
def test_denoising_unet_bf16_vs_oracle(lib, capsys, nf, depth, H, W):
    """bf16 denoising-sde network: full softmax Attention at mid_attn on the tensor cores (fullattn_mma_kernel, flash
    attention by mma.sync) - 1024 keys (the 256^2 / depth-4 mid level's token count), a ragged 520-key case (key masking,
    partial query block) and 4096 keys (the 512^2 count): per-layer report incl. the attention output."""
    dev = _dev()
    P = O.make_weights(3, 3, nf, depth, variant="denoising", seed=4)
    net = lib.DenoisingUNet(3, 3, nf, depth=depth, precision="bf16")
    net.load_state_dict(P, strict=True)
    net = net.to(dev)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(2, 3, H, W, generator=g) + torch.randn(2, 3, H, W, generator=g) * (50 / 255)
    yo, rows = _layer_report(net, P, x, None, 21, nf, depth, variant="denoising")
    y = net(x.to(dev), 21).cpu()
    with capsys.disabled():
        print("\nper-layer bf16 denoising-sde UNet vs fp32 oracle (nf=%d depth=%d, 2x3x%dx%d)" % (nf, depth, H, W))
        for key, dmax, rmax, rel in rows:
            if "mid" in key:
                print("  %-38s max|d| %.3e  max|ref| %.3e  rel-rms %.2e" % (key, dmax, rmax, rel))
    assert any(k == "mid_attn.full attention" for k, *_ in rows)
    for key, dmax, rmax, rel in rows:
        assert rel < 1.5e-2 and dmax < 3e-2 * rmax, (key, dmax, rmax, rel)
    assert (y - yo).abs().max().item() < 4e-2 * yo.abs().max().item()


def test_nafnet_w64_bf16_vs_oracle(lib):
    """ConditionalNAFNet at the Refusion width (w=64, 4 levels -> c=512 at H/8) on a 4-channel 64x64 latent, bf16 vs oracle."""
    dev = _dev()
    cfg = dict(img_channel=4, width=64, middle_blk_num=1, enc_blk_nums=[1, 1, 1, 4], dec_blk_nums=[1, 1, 1, 1])
    P = O.make_nafnet_weights(4, 64, 1, [1, 1, 1, 4], [1, 1, 1, 1], seed=6)
    g = torch.Generator().manual_seed(8)
    lq = torch.rand(2, 4, 64, 64, generator=g)
    x = lq + torch.randn(lq.shape, generator=g) * (50 / 255)
    yo = O.nafnet_forward(P, x, lq, 33, 64, [1, 1, 1, 4], 1, [1, 1, 1, 1], latent=True)
    for prec, tol in (("fp32", 1e-4), ("bf16", 2e-2 * yo.abs().max().item())):
        net = lib.ConditionalNAFNet(latent=True, precision=prec, **cfg)
        net.load_state_dict(P, strict=True)
        net = net.to(dev)
        y = net(x.to(dev), lq.to(dev), 33).cpu()
        assert (y - yo).abs().max().item() < tol, (prec, (y - yo).abs().max().item(), tol)


from _gpu_chain_helpers import _chain_pair, _drift_line  # noqa: E402


def test_bf16_chain_drift_report(lib, capsys):
    """Drift of a full T=100 chain in bf16 perf mode against the fp32 parity mode (itself within 1e-3 of the reference,
    test_chain_fp32_vs_reference), same x_T and z, 1x3x256x256, nf=64 depth=4 - reported, and bounded loosely:
    (a) the raw random-weight chain (expansive by 1/eps = 200x: a worst case no trained model shows), relative to |x0|;
    (b) the contractive, analytic-noise-assisted chain (see _chain_pair): bf16 must stay within 40 dB of fp32."""
    raw = _chain_pair(lib, ("fp32", "bf16"), assisted=False)
    ast = _chain_pair(lib, ("fp32", "bf16"), assisted=True)
    l1, d1, p1, ps1 = _drift_line("T=100 raw random-weight chain, bf16 vs fp32", raw["bf16"], raw["fp32"])
    l2, d2, p2, ps2 = _drift_line("T=100 assisted (contractive) chain, bf16 vs fp32", ast["bf16"], ast["fp32"])
    with capsys.disabled():
        print("\n" + l1 + "\n" + l2)
    assert torch.isfinite(raw["bf16"]).all() and d1.abs().max().item() < 0.1 * p1
    assert torch.isfinite(ast["bf16"]).all() and ps2 > 40.0
