"""The fp32-accurate tensor-core mode (precision="fp32x3": fp32 storage; every conv = three tf32 wgmma passes
over hi/lo split operands, conv_tc.cu MODE 3) against the same references and the SAME bounds as the fp32 SIMT parity mode:
convs 2e-5 (summation order + the 2^-21 split residue), network forwards 1e-4, full chains the north-star 1e-3 max-abs."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import irsde_oracle as O


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def _maxdiff(a, b):
    return (a.detach().float().cpu() - b.detach().float().cpu()).abs().max().item()


@pytest.fixture(scope="module")
def lib():
    import irsde_b200
    return irsde_b200


@pytest.fixture(scope="module")
def scratch_ctx(lib):
    _dev()
    return lib._lib.Context(3, 3, 8, 2, lib._lib.NET_CONDITIONAL, lib._lib.PREC_FP32, 0)


def _conv(lib, ctx, x, w, bias, res, stride, pad, up, silu):
    B, Cin, H, W = x.shape
    Cout, _, KH, KW = w.shape
    Ho = (H * (2 if up else 1) + 2 * pad - KH) // stride + 1
    Wo = (W * (2 if up else 1) + 2 * pad - KW) // stride + 1
    y = torch.empty(B, Cout, Ho, Wo, device=x.device)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    rc = ctx.L.irsde_conv2d_ex(ctx.h, 2, p(x.contiguous()), p(w.contiguous()), p(bias), p(res), p(y), B, Cin, H, W, Cout, KH, KW,
                               stride, pad, 1 if up else 0, 1 if silu else 0, 0,
                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    lib._lib.check(rc, ctx.h)
    torch.cuda.synchronize()
    return y


CASES = [
    # name, B, Cin, H, W, Cout, K, stride, pad, up, bias, silu, residual
    ("1x1 single chunk", 1, 32, 16, 16, 32, 1, 1, 0, False, False, False, False),
    ("3x3 ragged Cin/Cout, partial tiles", 2, 72, 10, 12, 40, 3, 1, 1, False, True, True, True),
    ("3x3 several K chunks, two N tiles", 1, 136, 9, 7, 200, 3, 1, 1, False, False, False, False),
    ("4x4 s2 space-to-depth planes", 2, 64, 16, 24, 128, 4, 2, 1, False, True, False, False),
    ("nearest x2 + 3x3 phases", 2, 128, 8, 12, 64, 3, 1, 1, True, True, False, False),
    ("head Cout=3 fp32 NCHW epilogue", 2, 64, 16, 24, 3, 3, 1, 1, False, True, False, False),
    ("to_qkv-like tiny K", 1, 8, 20, 28, 384, 1, 1, 0, False, False, False, False),
    # benchmark shapes, >= 2 x 132 tiles per launch: persistent multi-tile loop + segmented accumulation in MODE 3
    ("ups.0 block1 3x3 1536->1024 @32^2", 5, 1536, 32, 32, 1024, 3, 1, 1, False, False, True, False),
    ("downs.0 block 3x3 64->64 @256^2", 1, 64, 256, 256, 64, 3, 1, 1, False, False, True, True),
    ("ups.3 block1 3x3 192->128 @256^2", 1, 192, 256, 256, 128, 3, 1, 1, False, False, True, False),
    ("Downsample 4x4 s2 64->128 @256^2", 3, 64, 256, 256, 128, 4, 2, 1, False, True, False, False),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_fp32x3_vs_torch_fp32(lib, scratch_ctx, case):
    name, B, Cin, H, W, Cout, K, s, p, up, hb, silu, has_res = case
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(len(name) + Cin + Cout)
    x = torch.randn(B, Cin, H, W, generator=g, device=dev)
    w = torch.randn(Cout, Cin, K, K, generator=g, device=dev) / (Cin * K * K) ** 0.5
    b = torch.randn(Cout, generator=g, device=dev) if hb else None
    Ho = (H * (2 if up else 1) + 2 * p - K) // s + 1
    Wo = (W * (2 if up else 1) + 2 * p - K) // s + 1
    res = torch.randn(B, Cout, Ho, Wo, generator=g, device=dev) if has_res else None
    y = _conv(lib, scratch_ctx, x, w, b, res, s, p, up, silu)
    xin = F.interpolate(x, scale_factor=2, mode="nearest") if up else x
    ref = F.conv2d(xin.double(), w.double(), b.double() if hb else None, stride=s, padding=p)   # fp64: the exact answer
    if silu:
        ref = F.silu(ref)
    if res is not None:
        ref = ref + res.double()
    ref32 = F.conv2d(xin, w, b, stride=s, padding=p)
    if silu:
        ref32 = F.silu(ref32)
    if res is not None:
        ref32 = ref32 + res
    scale = ref.abs().max().item()
    err = (y.double() - ref).abs().max().item()
    err32 = (ref32.double() - ref).abs().max().item()            # what plain fp32 (cuDNN, TF32 off) gets on the same problem
    assert err <= max(2e-5 * scale, 8 * err32), (name, err, err32, scale)


def _net(lib, g, variant="conditional"):
    dev = _dev()
    cls = lib.ConditionalUNet if variant == "conditional" else lib.DenoisingUNet
    net = cls(3, 3, g["nf"], depth=g["depth"], precision="fp32x3")
    net.load_state_dict(g["state"], strict=True)
    return net.to(dev).eval()


def test_unet_forward_fp32x3_vs_reference(lib, golden):
    dev = _dev()
    g = golden["unet_cond"]
    net = _net(lib, g)
    y = net(g["xt"].to(dev), g["cond"].to(dev), g["t_int"])
    assert _maxdiff(y, g["y_int"]) < 1e-4            # the reference's own output (ragged 18x27 -> reflect pad)
    assert _maxdiff(net(g["xt"].to(dev), g["cond"].to(dev), g["t_vec"]), g["y_vec"]) < 1e-4
    ops = net.plan_ops(g["xt"].shape[0], g["xt"].shape[2], g["xt"].shape[3], dev)
    cats = [c for _, _, c in ops]
    assert cats.count(0) >= 40 and cats.count(1) <= 2   # convs run on the tensor-core engine (only the 7x7 stem stays SIMT)
    gd = golden["unet_dsde"]
    netd = _net(lib, gd, variant="denoising")
    assert _maxdiff(netd(gd["x"].to(dev), gd["t_int"]), gd["y"]) < 1e-4


@pytest.mark.parametrize("mode", ["sde", "ode", "posterior"])
def test_chain_fp32x3_vs_reference(lib, golden, mode):
    """Full T=20 chain and the partial T=5 chain against the reference's result, same z: the north-star 1e-3 max-abs."""
    dev = _dev()
    g, u = golden["irsde_chain"], golden["unet_cond"]
    net = _net(lib, u)
    sde = lib.IRSDE(g["args"][0], g["args"][1], schedule=g["args"][2], eps=g["args"][3], device=dev)
    sde.set_model(net)
    sde.set_mu(g["lq"].to(dev))
    c = g["chains"][mode]
    for graph in (True, False):
        sde.use_graph = graph
        d = _maxdiff(getattr(sde, "reverse_" + mode)(g["xT"].to(dev), zs=c["zs"].to(dev)), c["x0"])
        assert d < 1e-3, (mode, graph, d)
    assert _maxdiff(getattr(sde, "reverse_" + mode)(g["xT"].to(dev), T=5, zs=c["zs"].to(dev)), c["x0_T5"]) < 1e-3


def test_dsde_and_nafnet_fp32x3(lib, golden):
    dev = _dev()
    g = golden["unet_dsde"]
    net = _net(lib, g, variant="denoising")
    sde = lib.DenoisingSDE(g["args"][0], g["args"][1], schedule=g["args"][2], device=dev)
    sde.set_model(net)
    T = sde.get_optimal_timestep(25)
    assert _maxdiff(sde.reverse_sde(g["x"].to(dev), T=T, zs=g["zs"].to(dev)), g["x0_sde"]) < 1e-3
    assert _maxdiff(sde.reverse_ode(g["x"].to(dev), T=T), g["x0_ode"]) < 1e-3
    import os
    gn = torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_golden_nafnet.pt"), weights_only=True)["nafnet_latent"]
    naf = lib.ConditionalNAFNet(latent=gn["latent"], precision="fp32x3", **gn["cfg"])
    naf.load_state_dict(gn["state"], strict=True)
    naf = naf.to(dev)
    assert _maxdiff(naf(gn["x"].to(dev), gn["cond"].to(dev), gn["t_int"]), gn["y"]) < 1e-4


def test_nf64_chain_fp32x3_vs_fp32_and_oracle(lib, capsys):
    """BASELINE config 2's network (nf=64, depth=4) at 256x256: one forward vs the CPU oracle (1e-4), then a T=100 chain vs
    the fp32 SIMT parity mode, same x_T and z.  Random weights make the chain expand every difference by ~1/eps = 200x
    (tests/test_gpu_bench_shapes.py::_chain_pair), so the two fp32-accurate modes are compared relative to |x0| (<= 1e-4),
    and on the contractive analytic-noise-assisted chain at the absolute north-star bound 1e-3."""
    from _gpu_chain_helpers import _chain_pair, _drift_line
    dev = _dev()
    nf, depth = 64, 4
    P = O.make_weights(3, 3, nf, depth, seed=0)
    net = lib.ConditionalUNet(3, 3, nf, depth=depth, precision="fp32x3")
    net.load_state_dict(P, strict=True)
    net = net.to(dev)
    g = torch.Generator().manual_seed(1234)
    cond = torch.rand(1, 3, 256, 256, generator=g)
    xt = cond + torch.randn(1, 3, 256, 256, generator=g) * (10 / 255)
    yo = O.unet_forward(P, xt, cond, 57, nf, depth)
    d_fwd = _maxdiff(net(xt.to(dev), cond.to(dev), 57), yo)
    # per-layer relative RMS error of both fp32-accurate modes against the CPU oracle
    from test_gpu_bench_shapes import _layer_report
    _, rows3 = _layer_report(net, P, xt, cond, 57, nf, depth)
    del net
    net1 = lib.ConditionalUNet(3, 3, nf, depth=depth, precision="fp32")
    net1.load_state_dict(P, strict=True)
    net1 = net1.to(dev)
    _, rows1 = _layer_report(net1, P, xt, cond, 57, nf, depth)
    del net1
    with capsys.disabled():
        print("\nper-layer rel-rms vs fp32 CPU oracle (nf=64 depth=4, 1x3x256x256): fp32 SIMT | fp32x3 tensor-core")
        for (k1, _, _, r1), (k3, _, _, r3) in zip(rows1, rows3):
            if "block2" in k1 or "3." in k1 or "norm+res" in k1:
                print("  %-38s %.2e | %.2e" % (k1, r1, r3))
    raw = _chain_pair(lib, ("fp32", "fp32x3"), assisted=False)
    ast = _chain_pair(lib, ("fp32", "fp32x3"), assisted=True)
    l1, d1, p1, _ = _drift_line("T=100 raw random-weight chain, fp32x3 vs fp32", raw["fp32x3"], raw["fp32"])
    l2, d2, p2, _ = _drift_line("T=100 assisted (contractive) chain, fp32x3 vs fp32", ast["fp32x3"], ast["fp32"])
    with capsys.disabled():
        print("\nnf=64 forward fp32x3 vs oracle: max|d| %.3e (max|ref| %.3g)\n%s\n%s" % (d_fwd, yo.abs().max().item(), l1, l2))
    assert d_fwd < 1e-4
    assert d1.abs().max().item() < 1e-4 * max(p1, 1.0)
    assert d2.abs().max().item() < 1e-3
