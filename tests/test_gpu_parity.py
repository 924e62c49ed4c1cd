"""GPU parity tests (H100): the CUDA path, called through the C ABI, against the CPU oracle and the
golden outputs of the imported reference.  Tolerances are stated per test.

fp32 "parity mode" is held to the north-star bound (1e-3 max-abs per pixel) with large margin;
bf16 "perf mode" is judged per network forward / teacher-forced step (SURVEY 0: the chain amplifies
a 1e-6 perturbation to ~5e-4, so bf16 cannot meet 1e-3 end to end by construction).
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import irsde_oracle as O


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
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


def _conv2d(lib, ctx, engine, x, w, bias, stride, pad, up, silu):
    dev = _dev()
    xg, wg = x.to(dev).contiguous(), w.to(dev).contiguous()
    bg = bias.to(dev).contiguous() if bias is not None else None
    B, Cin, H, W = x.shape
    Cout, _, KH, KW = w.shape
    Ho = (H * (2 if up else 1) + 2 * pad - KH) // stride + 1
    Wo = (W * (2 if up else 1) + 2 * pad - KW) // stride + 1
    y = torch.empty(B, Cout, Ho, Wo, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    rc = ctx.L.irsde_conv2d(ctx.h, engine, p(xg), p(wg), p(bg), p(y), B, Cin, H, W, Cout, KH, KW, stride, pad,
                            1 if up else 0, 1 if silu else 0, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    lib._lib.check(rc, ctx.h)
    torch.cuda.synchronize()
    return y.cpu()


def _conv_ref(x, w, bias, stride, pad, up, silu):
    if up:
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    y = F.conv2d(x, w, bias, stride=stride, padding=pad)
    return F.silu(y) if silu else y


def test_sde_steps_bitexact(lib, golden):
    """Fused update kernel vs the reference's own step outputs: same op order, no FMA contraction."""
    dev = _dev()
    g = golden["irsde_steps"]
    sde = lib.IRSDE(*g["args"][:2], schedule=g["args"][2], eps=g["args"][3], device=dev)
    x, mu, noise = g["x"].to(dev), g["mu"].to(dev), g["noise"].to(dev)
    for st in g["steps"]:
        t, z = st["t"], st["z"].to(dev)
        for mode, key in ((lib._lib.MODE_SDE, "sde"), (lib._lib.MODE_ODE, "ode"), (lib._lib.MODE_POSTERIOR, "posterior")):
            out = sde._native_step(mode, x, mu, noise, z if key != "ode" else None, t)
            d = _maxdiff(out, st[key])
            assert d <= 2e-6, (key, t, d)  # <= 1 ulp of |x|~4 (GPU division/transcendental-free path)
    g = golden["dsde_steps"]
    dsde = lib.DenoisingSDE(*g["args"][:2], schedule=g["args"][2], device=dev)
    x, noise = g["x"].to(dev), g["noise"].to(dev)
    for st in g["steps"]:
        z = st["z"].to(dev)
        assert _maxdiff(dsde._native_step(lib._lib.MODE_DSDE_SDE, x, None, noise, z, st["t"]), st["sde"]) <= 2e-6
        assert _maxdiff(dsde._native_step(lib._lib.MODE_DSDE_ODE, x, None, noise, None, st["t"]), st["ode"]) <= 2e-6


def _net(lib, g, precision="fp32", variant="conditional", force_simt=False):
    dev = _dev()
    cls = lib.ConditionalUNet if variant == "conditional" else lib.DenoisingUNet
    net = cls(3, 3, g["nf"], depth=g["depth"], precision=precision, force_simt=force_simt)
    net.load_state_dict(g["state"], strict=True)
    return net.to(dev).eval()


def test_unet_forward_fp32(lib, golden):
    g = golden["unet_cond"]
    net = _net(lib, g)
    dev = _dev()
    y = net(g["xt"].to(dev), g["cond"].to(dev), g["t_int"])
    assert y.shape == g["y_int"].shape
    assert _maxdiff(y, g["y_int"]) < 1e-4            # vs the reference's own output (ragged 18x27 -> reflect pad)
    y2 = net(g["xt"].to(dev), g["cond"].to(dev), g["t_vec"])
    assert _maxdiff(y2, g["y_vec"]) < 1e-4           # per-image timesteps
    yo = O.unet_forward(g["state"], g["xt"], g["cond"], g["t_int"], g["nf"], g["depth"])
    assert _maxdiff(y, yo) < 1e-4                    # vs the oracle


def test_unet_forward_fp32_wider(lib):
    """Larger widths / depth 3 / several K tiles, random weights, CUDA vs oracle."""
    dev = _dev()
    P = O.make_weights(3, 3, 16, 3, seed=5)
    net = lib.ConditionalUNet(3, 3, 16, depth=3, precision="fp32")
    net.load_state_dict(P, strict=True)
    net = net.to(dev)
    g = torch.Generator().manual_seed(9)
    xt, cond = torch.rand(2, 3, 40, 24, generator=g), torch.rand(2, 3, 40, 24, generator=g)
    y = net(xt.to(dev), cond.to(dev), 17)
    yo = O.unet_forward(P, xt, cond, 17, 16, 3)
    assert _maxdiff(y, yo) < 2e-4


def test_unet_denoising_variant_fp32(lib, golden):
    g = golden["unet_dsde"]
    net = _net(lib, g, variant="denoising")
    y = net(g["x"].to(_dev()), g["t_int"])
    assert _maxdiff(y, g["y"]) < 1e-4


@pytest.mark.parametrize("mode", ["sde", "ode", "posterior"])
@pytest.mark.parametrize("graph", [True, False])
def test_chain_fp32_vs_reference(lib, golden, mode, graph):
    """Full T=20 chain (and the partial T=5 chain) against the reference's result, same z.
    Bound: the north-star 1e-3 max-abs."""
    dev = _dev()
    g, u = golden["irsde_chain"], golden["unet_cond"]
    net = _net(lib, u)
    sde = lib.IRSDE(g["args"][0], g["args"][1], schedule=g["args"][2], eps=g["args"][3], device=dev)
    sde.use_graph = graph
    sde.set_model(net)
    sde.set_mu(g["lq"].to(dev))
    c = g["chains"][mode]
    x0 = getattr(sde, "reverse_" + mode)(g["xT"].to(dev), zs=c["zs"].to(dev))
    assert _maxdiff(x0, c["x0"]) < 1e-3
    x5 = getattr(sde, "reverse_" + mode)(g["xT"].to(dev), T=5, zs=c["zs"].to(dev))
    assert _maxdiff(x5, c["x0_T5"]) < 1e-3


def test_chain_stepwise_equals_fused(lib, golden):
    """Generic python loop (noise_fn + step kernel) == library chain, bit for bit (same kernels)."""
    dev = _dev()
    g, u = golden["irsde_chain"], golden["unet_cond"]
    net = _net(lib, u)
    sde = lib.IRSDE(g["args"][0], g["args"][1], schedule=g["args"][2], eps=g["args"][3], device=dev)
    sde.set_model(net)
    sde.set_mu(g["lq"].to(dev))
    zs = g["chains"]["sde"]["zs"].to(dev)
    a = sde.reverse_sde(g["xT"].to(dev), zs=zs)
    x = g["xT"].to(dev).clone()
    for i, t in enumerate(reversed(range(1, sde.T + 1))):
        x = sde._native_step(lib._lib.MODE_SDE, x, sde.mu, sde.noise_fn(x, t), zs[i], t)
    assert torch.equal(a, x)


def test_dsde_chain_fp32(lib, golden):
    dev = _dev()
    g = golden["unet_dsde"]
    net = _net(lib, g, variant="denoising")
    sde = lib.DenoisingSDE(g["args"][0], g["args"][1], schedule=g["args"][2], device=dev)
    sde.set_model(net)
    T = sde.get_optimal_timestep(25)
    assert int(T) == g["Tstar"]                      # integer work: bit-exact
    zs = g["zs"].to(dev)
    assert _maxdiff(sde.reverse_sde(g["x"].to(dev), T=T, zs=zs), g["x0_sde"]) < 1e-3
    assert _maxdiff(sde.reverse_ode(g["x"].to(dev), T=T), g["x0_ode"]) < 1e-3


def test_sharded_equals_unsharded(lib, golden):
    """Batch slices processed independently == full batch (bit-identical): the multi-GPU partition."""
    dev = _dev()
    u = golden["unet_cond"]
    net = _net(lib, u)
    sde = lib.IRSDE(10, 10, schedule="cosine", eps=0.005, device=dev)
    sde.set_model(net)
    g = torch.Generator().manual_seed(4)
    lq = torch.rand(3, 3, 16, 16, generator=g).to(dev)
    xT = lq + torch.randn(3, 3, 16, 16, generator=g).to(dev) * sde.max_sigma
    zs = torch.randn(10, 3, 3, 16, 16, generator=g).to(dev)
    sde.set_mu(lq)
    full = sde.reverse_sde(xT, zs=zs)
    parts = []
    for r in range(2):
        lo, hi = lib.shard_range(3, r, 2)
        sde.set_mu(lq[lo:hi])
        parts.append(sde.reverse_sde(xT[lo:hi], zs=zs[:, lo:hi]))
    assert torch.equal(full, torch.cat(parts))


def test_philox_noise_statistics(lib):
    dev = _dev()
    sde = lib.IRSDE(10, 4, device=dev)
    net = lib.ConditionalUNet(3, 3, 8, depth=2).to(dev)
    sde.set_model(net)
    ctx = sde._ctx_for(torch.zeros(1, device=dev))
    mu = torch.zeros(1 << 20, device=dev)
    out = torch.empty_like(mu)
    lib._lib.check(ctx.L.irsde_noise_state(ctx.h, ctypes.c_void_p(mu.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                           mu.numel(), 123, None), ctx.h)
    torch.cuda.synchronize()
    z = out / sde.max_sigma
    assert abs(z.mean().item()) < 5e-3 and abs(z.std().item() - 1) < 5e-3
    assert abs((z ** 4).mean().item() - 3) < 0.1


# ------------------------------------------------------------------------------------------------
# bf16 perf mode
# ------------------------------------------------------------------------------------------------
TC_CASES = [
    # B, Cin, H, W, Cout, K, stride, pad, up, bias, silu
    (1, 64, 16, 16, 64, 1, 1, 0, False, False, False),   # single tap, single K chunk, BN=64
    (1, 64, 16, 16, 64, 3, 1, 1, False, False, False),   # 9 taps: TMA OOB zero padding
    (2, 128, 16, 32, 128, 3, 1, 1, False, True, True),   # 2 K chunks, BN=128, bias+SiLU epilogue
    (1, 192, 8, 8, 256, 3, 1, 1, False, False, False),   # BN=256, 3 K chunks, 8x8 image (BW=8)
    (2, 72, 10, 12, 40, 3, 1, 1, False, True, False),    # ragged: Cin%64!=0, Cout%32!=0, partial tiles
    (2, 64, 16, 24, 128, 4, 2, 1, False, True, False),   # downsample over space-to-depth planes
    (2, 128, 8, 12, 64, 3, 1, 1, True, True, False),     # upsample phases with pre-summed weights
    (1, 8, 20, 28, 384, 1, 1, 0, False, False, False),   # to_qkv at nf=8: tiny K, 2 N tiles
    (2, 6, 20, 28, 64, 7, 1, 3, False, False, False),    # 7x7 stem as 7 row-taps (overlapping-stride TMA view)
    (1, 3, 9, 13, 16, 7, 1, 3, False, False, False),     # stem of the denoising variant (Cin=3), ragged size
    (2, 64, 16, 24, 3, 3, 1, 1, False, True, False),     # head: Cout=3, fp32 NCHW straight from the epilogue
]


@pytest.mark.parametrize("case", TC_CASES)
def test_conv_tcgen05(lib, scratch_ctx, case):
    """Tensor-core (wgmma) tap-GEMM vs fp32 conv on bf16-rounded operands (fp32 accumulation => only the output
    rounding to bf16 and summation order differ): tolerance 2^-8 relative to the output scale."""
    B, Cin, H, W, Cout, K, s, p, up, hb, silu = case
    g = torch.Generator().manual_seed(sum(case[:6]))
    x = torch.randn(B, Cin, H, W, generator=g).bfloat16().float()
    w = (torch.randn(Cout, Cin, K, K, generator=g) / (Cin * K * K) ** 0.5)
    b = torch.randn(Cout, generator=g) if hb else None
    y = _conv2d(lib, scratch_ctx, 1, x, w, b, s, p, up, silu)
    if up:
        # the engine pre-sums weights per output phase before rounding to bf16; compare to the fp32 conv
        ref = _conv_ref(x, w, b, s, p, up, silu)
        tol = 3e-2
    else:
        ref = _conv_ref(x, w.bfloat16().float(), b, s, p, up, silu)
        tol = 1.5e-2
    scale = ref.abs().max().item()
    assert _maxdiff(y, ref) < tol * max(scale, 1.0), (_maxdiff(y, ref), scale)


@pytest.mark.parametrize("force_simt", [True, False])
def test_unet_forward_bf16(lib, golden, force_simt):
    """bf16 perf mode (force_simt=True: same bf16 storage through the SIMT engine; False: tensor cores)
    vs the fp32 oracle on one forward: relative error of a bf16 pipeline (~1e-2 of the output scale)."""
    dev = _dev()
    P = O.make_weights(3, 3, 16, 3, seed=5)
    net = lib.ConditionalUNet(3, 3, 16, depth=3, precision="bf16", force_simt=force_simt)
    net.load_state_dict(P, strict=True)
    net = net.to(dev)
    g = torch.Generator().manual_seed(9)
    xt, cond = torch.rand(2, 3, 40, 24, generator=g), torch.rand(2, 3, 40, 24, generator=g)
    y = net(xt.to(dev), cond.to(dev), 17)
    yo = O.unet_forward(P, xt, cond, 17, 16, 3)
    scale = yo.abs().max().item()
    assert _maxdiff(y, yo) < 4e-2 * scale, (_maxdiff(y, yo), scale)


def test_step_bf16_teacher_forced(lib, golden):
    """Per-step bound for perf mode: x_{t-1} from the bf16 network vs the fp32 oracle step, same x_t."""
    dev = _dev()
    P = O.make_weights(3, 3, 16, 3, seed=5)
    net = lib.ConditionalUNet(3, 3, 16, depth=3, precision="bf16")
    net.load_state_dict(P, strict=True)
    net = net.to(dev)
    sde = lib.IRSDE(10, 100, schedule="cosine", eps=0.005, device=dev)
    sde.set_model(net)
    sc = O.Schedule(10, 100, "cosine", 0.005)
    g = torch.Generator().manual_seed(2)
    lq = torch.rand(1, 3, 32, 32, generator=g)
    xt = lq + torch.randn(1, 3, 32, 32, generator=g) * sc.max_sigma
    z = torch.randn(1, 3, 32, 32, generator=g)
    sde.set_mu(lq.to(dev))
    for t in (100, 50, 1):
        eps_o = O.unet_forward(P, xt, lq, t, 16, 3)
        ref = O.irsde_sde_step(sc, xt, lq, eps_o, z, t)
        out = sde._native_step(lib._lib.MODE_SDE, xt.to(dev), sde.mu, sde.noise_fn(xt.to(dev), t), z.to(dev), t)
        assert _maxdiff(out, ref) < 1e-3, (t, _maxdiff(out, ref))


# ------------------------------------------------------------------------------------------------
# ConditionalNAFNet (Refusion score network)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden_naf():
    import os
    return torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_golden_nafnet.pt"), weights_only=True)


@pytest.mark.parametrize("key", ["nafnet", "nafnet_latent"])
def test_nafnet_forward_fp32(lib, golden_naf, key):
    """fp32 parity mode vs the reference's own output (zero pad 18x23 -> 20x24, scalar and per-image t)."""
    dev = _dev()
    g = golden_naf[key]
    c = g["cfg"]
    net = lib.ConditionalNAFNet(latent=g["latent"], precision="fp32", **c)
    assert list(net.state_dict().keys()) == list(g["state"].keys())
    net.load_state_dict(g["state"], strict=True)
    net = net.to(dev)
    y = net(g["x"].to(dev), g["cond"].to(dev), g["t_int"])
    assert _maxdiff(y, g["y"]) < 1e-4
    yv = net(g["x"].to(dev), g["cond"].to(dev), g["t_vec"])
    assert _maxdiff(yv, g["y_vec"]) < 1e-4


def test_nafnet_chain_fp32_and_bf16(lib):
    """Refusion-style chain (reverse_sde through NAFNet) vs the oracle: fp32 <= 1e-3; bf16 forward <= 4% of scale."""
    dev = _dev()
    cfg = dict(img_channel=4, width=16, middle_blk_num=1, enc_blk_nums=[1, 1], dec_blk_nums=[1, 1])
    P = O.make_nafnet_weights(4, 16, 1, [1, 1], [1, 1], seed=3)
    g = torch.Generator().manual_seed(8)
    lq = torch.rand(2, 4, 24, 32, generator=g)
    T = 6
    sc = O.Schedule(50, T, "cosine", 0.005)
    xT = lq + torch.randn(lq.shape, generator=g) * sc.max_sigma
    zs = torch.randn((T,) + tuple(lq.shape), generator=g)
    fn = lambda x, t: O.nafnet_forward(P, x, lq, t, 16, [1, 1], 1, [1, 1], latent=True)
    ref = O.reverse_chain(sc, fn, xT, lq, zs, "sde")
    net = lib.ConditionalNAFNet(latent=True, precision="fp32", **cfg)
    net.load_state_dict(P, strict=True)
    net = net.to(dev)
    sde = lib.IRSDE(50, T, schedule="cosine", eps=0.005, device=dev)
    sde.set_model(net)
    sde.set_mu(lq.to(dev))
    x0 = sde.reverse_sde(xT.to(dev), zs=zs.to(dev))
    assert _maxdiff(x0, ref) < 1e-3
    netb = lib.ConditionalNAFNet(latent=True, precision="bf16", **cfg)
    netb.load_state_dict(P, strict=True)
    netb = netb.to(dev)
    yo = fn(xT, 3)
    yb = netb(xT.to(dev), lq.to(dev), 3)
    assert _maxdiff(yb, yo) < 4e-2 * yo.abs().max().item()


# ------------------------------------------------------------------------------------------------
# BASELINE.json full-size workload (config 2: 8x3x256x256, nf=64 depth=4): size-independent properties
# ------------------------------------------------------------------------------------------------
def test_full_size_properties_bf16(lib):
    """At the benchmark size the oracle is too slow, so check properties that do not need it:
    (1) graph replay == eager launch, bit for bit; (2) run-to-run determinism; (3) batch-sharded (the multi-GPU
    partition) == unsharded, bit for bit; (4) finite outputs; (5) with eps-hat from the analytic noise of a known x0
    the sampler update itself contracts toward x0 (sampler-only chain, no network)."""
    dev = _dev()
    torch.manual_seed(0)
    net = lib.ConditionalUNet(3, 3, 64, depth=4, precision="bf16").to(dev)
    sde = lib.IRSDE(10, 100, schedule="cosine", eps=0.005, device=dev)
    sde.set_model(net)
    g = torch.Generator().manual_seed(1234)
    lq = torch.rand(8, 3, 256, 256, generator=g).to(dev)
    xT = lq + torch.randn(8, 3, 256, 256, generator=g).to(dev) * sde.max_sigma
    T = 3
    zs = torch.randn(T, 8, 3, 256, 256, generator=g).to(dev)
    sde.set_mu(lq)
    sde.use_graph = True
    a = sde.reverse_sde(xT, T=T, zs=zs)
    b = sde.reverse_sde(xT, T=T, zs=zs)
    sde.use_graph = False
    c = sde.reverse_sde(xT, T=T, zs=zs)
    assert torch.isfinite(a).all()
    assert torch.equal(a, b) and torch.equal(a, c)
    parts = []
    for r in range(2):
        lo, hi = lib.shard_range(8, r, 2)
        sde.set_mu(lq[lo:hi])
        parts.append(sde.reverse_sde(xT[lo:hi], T=T, zs=zs[:, lo:hi]))
    assert torch.equal(a, torch.cat(parts))
    # sampler-only chain with the analytic noise (sde_utils.py:231-232): converges to x0
    sde.set_mu(lq)
    x0 = torch.rand(8, 3, 256, 256, generator=g).to(dev)
    x = sde.mu + (x0 - sde.mu) * torch.exp(-sde.thetas_cumsum[100] * sde.dt) + torch.randn_like(x0) * sde.sigma_bars[100]
    for t in reversed(range(1, 101)):
        eps_true = sde.get_real_noise(x, x0, t)
        x = sde._native_step(lib._lib.MODE_POSTERIOR, x, sde.mu, eps_true, torch.randn_like(x), t)
    assert _maxdiff(x, x0) < 1e-3


# ------------------------------------------------------------------------------------------------
# Refusion latent autoencoder UNet.encode / decode
# ------------------------------------------------------------------------------------------------
def test_latent_unet_fp32_vs_reference(lib):
    import os
    dev = _dev()
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_golden_latent.pt"), weights_only=True)
    net = lib.UNet(precision="fp32", **g["cfg"])
    assert list(net.state_dict().keys()) == list(g["state"].keys())
    net.load_state_dict(g["state"], strict=True)
    net = net.to(dev)
    z, h = net.encode(g["x"].to(dev))
    assert z.shape == g["z"].shape and _maxdiff(z, g["z"]) < 1e-4   # ragged 21x30 -> reflect pad 24x32, latent 12x16
    assert _maxdiff(net.decode(g["z2"].to(dev), h), g["y"]) < 1e-4   # decode of a perturbed latent with the LQ's skips
    assert _maxdiff(net(g["x"].to(dev)), g["y_id"]) < 1e-4
    _, h2 = net.encode(g["x"].to(dev))
    with pytest.raises(RuntimeError):      # the skips of `h` were overwritten by the later encode: must not decode silently
        net.decode(g["z2"].to(dev), h)
    assert _maxdiff(net.decode(g["z2"].to(dev), h2), g["y"]) < 1e-4


def test_latent_unet_bf16_and_real_architecture(lib):
    """The shipped checkpoint's architecture (ch=8, ch_mult=[4,8,8,16], embed 8) with random weights: fp32 vs oracle
    <= 2e-4, bf16 (tensor-core path) within 4 % of the output scale."""
    dev = _dev()
    cfg = dict(in_ch=3, out_ch=3, ch=8, ch_mult=[4, 8, 8, 16], embed_dim=8)
    P = O.make_latent_unet_weights(3, 3, 8, [4, 8, 8, 16], 8, seed=2)
    g = torch.Generator().manual_seed(3)
    x = torch.rand(2, 3, 70, 90, generator=g)
    zo, ho = O.latent_unet_encode(P, x, cfg["ch_mult"])
    yo = O.latent_unet_decode(P, zo, ho, cfg["ch_mult"], 70, 90)
    for prec, tz, ty in (("fp32", 2e-4, 2e-4), ("bf16", 4e-2 * zo.abs().max().item(), 4e-2 * yo.abs().max().item())):
        net = lib.UNet(precision=prec, **cfg)
        net.load_state_dict(P, strict=True)
        net = net.to(dev)
        z, h = net.encode(x.to(dev))
        assert _maxdiff(z, zo) < tz, (prec, _maxdiff(z, zo))
        y = net.decode(zo.to(dev), h)
        assert _maxdiff(y, yo) < ty, (prec, _maxdiff(y, yo))


# ------------------------------------------------------------------------------------------------
# image helpers on the device (SURVEY 8 f-3): tensor2img / img2tensor / PSNR / SSIM
# ------------------------------------------------------------------------------------------------
def test_imaging_bit_exact_vs_reference(lib):
    import os
    import numpy as np
    dev = _dev()
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_golden_imaging.npz"))
    for k in "abc":
        t = torch.from_numpy(g["t_" + k]).to(dev)
        assert np.array_equal(lib.tensor2img(t), g["img_" + k])                    # uint8, BGR/HWC, .5 ties: bit exact
        assert np.array_equal(lib.tensor2img(t * 2 - 1, min_max=(-1, 1)), g["img11_" + k])
    x, y = g["x"], g["y"]
    assert np.array_equal(lib.imaging.img2tensor_device(x).cpu().numpy(), g["x_tensor"])
    assert lib.calculate_psnr(x, y) == float(g["psnr"])                            # exact integer sum -> same float64
    assert lib.calculate_psnr(x, y, crop_border=4) == float(g["psnr_crop4"])
    assert lib.calculate_psnr(x, x) == float("inf")
    assert abs(lib.calculate_ssim(x, y) - float(g["ssim"])) < 1e-10
    assert abs(lib.calculate_ssim(x, y, crop_border=4) - float(g["ssim_crop4"])) < 1e-10
    assert abs(lib.calculate_ssim(x[:, :, 0], y[:, :, 0]) - float(g["ssim_gray"])) < 1e-10
    with pytest.raises(ValueError):
        lib.calculate_ssim(x[:12, :12], y[:12, :12], crop_border=1)               # 10x10 after crop: no valid window


def test_imaging_batched_vs_oracle(lib):
    """Batch of 256x256 images (vectorised path) and a ragged 321x481 one: device == numpy oracle, bit for bit."""
    import numpy as np
    from oracle import imaging_oracle as IO
    dev = _dev()
    g = torch.Generator().manual_seed(5)
    t = torch.rand(4, 3, 256, 256, generator=g) * 1.2 - 0.1
    imgs = lib.imaging.tensor2img_device(t.to(dev))
    ref = np.stack([IO.tensor2img(t[i].numpy()) for i in range(4)])
    assert imgs.dtype == torch.uint8 and np.array_equal(imgs.cpu().numpy(), ref)
    back = lib.imaging.img2tensor_device(imgs)
    assert np.array_equal(back.cpu().numpy(), np.stack([IO.img2tensor(ref[i]) for i in range(4)]))
    other = torch.from_numpy(ref).roll(1, 0)
    se = lib.imaging.sqerr_device(imgs, other.to(dev), crop_border=3).cpu().numpy()
    for i in range(4):
        a, b = ref[i][3:-3, 3:-3].astype(np.int64), other[i].numpy()[3:-3, 3:-3].astype(np.int64)
        assert int(se[i]) == int(((a - b) ** 2).sum())
    noisy = np.clip(ref.astype(np.int32) + torch.randint(-9, 10, ref.shape, generator=g).numpy(), 0, 255).astype(np.uint8)
    ss = lib.imaging.ssim_device(ref, noisy).cpu().numpy()
    for i in range(4):
        assert abs(ss[i] - IO.calculate_ssim(ref[i], noisy[i])) < 1e-10
    r = torch.rand(3, 321, 481, generator=g)
    assert np.array_equal(lib.tensor2img(r.to(dev)), IO.tensor2img(r.numpy()))


# ------------------------------------------------------------------------------------------------
# per-image Philox + batched restoration front-end (SURVEY 8 f-2)
# ------------------------------------------------------------------------------------------------
def test_philox_is_keyed_per_image(lib):
    """In-kernel noise depends on (seed, image uid, t, element) only: batched == sharded == one at a time, bit for bit,
    also when an image's element count is not a multiple of 4 (Philox blocks straddle images)."""
    dev = _dev()
    torch.manual_seed(0)
    net = lib.ConditionalUNet(3, 3, 8, depth=2).to(dev)
    sde = lib.IRSDE(25, 6, eps=0.005, device=dev)
    sde.set_model(net)
    sde.rng, sde.seed_auto_increment, sde.seed = "philox", False, 11
    for (H, W) in ((12, 16), (9, 7)):            # 3*9*7 = 189 elements per image: not a multiple of 4
        lq = torch.rand(4, 3, H, W, device=dev)
        sde.image_base, sde.image_uids = 0, None
        xT = sde.noise_state(lq)
        sde.set_mu(lq)
        full = sde.reverse_sde(xT)
        assert (xT - lq).std().item() > 0.5 * sde.max_sigma
        assert not torch.equal(xT[0] - lq[0], xT[1] - lq[1])                       # images get different noise
        for lo, hi in ((0, 2), (2, 4), (1, 2), (3, 4)):
            sde.image_base = lo
            assert torch.equal(sde.noise_state(lq[lo:hi]), xT[lo:hi])
            sde.set_mu(lq[lo:hi])
            assert torch.equal(sde.reverse_sde(xT[lo:hi]), full[lo:hi])
        sde.image_base, sde.image_uids = 0, [3, 1]                                  # explicit uids: a re-ordered batch
        sel = torch.tensor([3, 1], device=dev)
        assert torch.equal(sde.noise_state(lq[sel]), xT[sel])
        sde.set_mu(lq[sel])
        assert torch.equal(sde.reverse_sde(xT[sel]), full[sel])
        sde.image_uids = None
    sde.seed = 12
    assert not torch.equal(sde.noise_state(lq), xT)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_restorer_batched_equals_single(lib, precision):
    """uint8 in -> uint8 out; mixed image sizes; any batch size gives the images of the one-at-a-time run, and those
    equal the hand-written sequence img2tensor -> noise_state -> reverse_sde -> tensor2img."""
    import numpy as np
    dev = _dev()
    torch.manual_seed(1)
    net = lib.ConditionalUNet(3, 3, 16, depth=2, precision=precision).to(dev)
    sde = lib.IRSDE(10, 5, eps=0.005, device=dev)
    sde.set_model(net)
    g = torch.Generator().manual_seed(2)
    shapes = [(24, 32), (16, 16), (24, 32), (24, 32), (16, 16), (24, 32)]
    imgs = [(torch.rand(h, w, 3, generator=g) * 255).to(torch.uint8).numpy() for h, w in shapes]
    one = lib.Restorer(sde, mode="sde", batch_size=1, seed=5).restore(imgs)
    for bs in (2, 4):
        many = lib.Restorer(sde, mode="sde", batch_size=bs, seed=5).restore(imgs)
        for a, b in zip(one, many):
            assert a.dtype == np.uint8 and a.shape == b.shape and np.array_equal(a, b)
    assert not np.array_equal(one[0], lib.Restorer(sde, mode="sde", batch_size=4, seed=6).restore(imgs)[0])
    # image 4 by hand
    sde.rng, sde.seed, sde.seed_auto_increment, sde.image_uids = "philox", 5, False, [4]
    lq = lib.imaging.img2tensor_device(imgs[4])[None]
    sde.set_mu(lq)
    x0 = sde.reverse_sde(sde.noise_state(lq))
    assert np.array_equal(lib.tensor2img(x0), one[4])
    sde.image_uids = None
    assert np.array_equal(lib.Restorer(sde, mode="ode", batch_size=3).restore(imgs)[2],
                          lib.Restorer(sde, mode="ode", batch_size=1).restore(imgs)[2])


# ------------------------------------------------------------------------------------------------
# context hygiene (round-1 advisor findings)
# ------------------------------------------------------------------------------------------------
def test_two_samplers_share_one_network(lib, golden):
    """The schedule / coefficient tables live in the MODEL's native context: two samplers with different T and max_sigma
    driving one network must each see their own tables, in any interleaving."""
    dev = _dev()
    net = _net(lib, golden["unet_cond"])
    g = torch.Generator().manual_seed(3)
    lq = torch.rand(1, 3, 16, 16, generator=g).to(dev)
    a, b = lib.IRSDE(10, 12, eps=0.005, device=dev), lib.IRSDE(30, 7, schedule="linear", eps=0.01, device=dev)
    outs = {}
    for name, sde in (("a", a), ("b", b), ("a2", a), ("b2", b)):
        sde.set_model(net)
        sde.set_mu(lq)
        xT = lq + 0.1
        zs = torch.randn(sde.T, 1, 3, 16, 16, generator=torch.Generator().manual_seed(5)).to(dev)
        outs[name] = sde.reverse_posterior(xT, zs=zs)
    assert torch.equal(outs["a"], outs["a2"]) and torch.equal(outs["b"], outs["b2"])
    assert not torch.equal(outs["a"], outs["b"])
    # and against the oracle, after the other sampler wrote last
    u = golden["unet_cond"]
    sc = O.Schedule(10, 12, "cosine", 0.005)
    zs = torch.randn(12, 1, 3, 16, 16, generator=torch.Generator().manual_seed(5))
    ref = O.reverse_chain(sc, lambda x, t: O.unet_forward(u["state"], x, lq.cpu(), t, u["nf"], u["depth"]), lq.cpu() + 0.1, lq.cpu(), zs,
                          "posterior")
    assert _maxdiff(outs["a2"], ref) < 1e-3


def test_scalar_mu_before_set_mu(lib):
    """IRSDE starts with mu = 0. (a float, sde_utils.py:88): the step functions broadcast it like the reference."""
    dev = _dev()
    sde = lib.IRSDE(10, 10, device=dev)
    x = torch.rand(1, 3, 8, 8, device=dev)
    score = torch.rand(1, 3, 8, 8, device=dev)
    out = sde.reverse_ode_step(x, score, 5)
    ref = x - (sde.thetas[5] * (0. - x) - 0.5 * sde.sigmas[5] ** 2 * score) * sde.dt.to(dev)
    assert _maxdiff(out, ref) < 1e-6


def test_plan_cache_is_bounded_and_trim(lib):
    """A loop over variable-size images must not grow device memory without limit: the plan cache keeps at most
    IRSDE_PLAN_CACHE_MAX (default 8) shapes; irsde_trim drops them all; results do not depend on cache state."""
    dev = _dev()
    torch.manual_seed(0)
    net = lib.ConditionalUNet(3, 3, 8, depth=2).to(dev)
    x = torch.rand(1, 3, 16, 16, device=dev)
    first = net(x, x, 3)
    ctx = net._ctx
    sizes = []
    for k in range(14):
        h = 16 + 4 * k
        net(torch.rand(1, 3, h, 20, device=dev), torch.rand(1, 3, h, 20, device=dev), 3)
        sizes.append(int(ctx.L.irsde_device_bytes(ctx.h)))
    assert sizes[-1] < sizes[7] * 2.5          # 14 ever-larger shapes, memory of <= 8 of them
    lib._lib.check(ctx.L.irsde_trim(ctx.h), ctx.h)
    assert int(ctx.L.irsde_device_bytes(ctx.h)) < sizes[0]
    assert torch.equal(net(x, x, 3), first)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_unet_ch_mult_variant(lib, precision):
    """The latent tasks' ConditionalUNet(in_nc, out_nc, nf, ch_mult): fp32 <= 1e-4 vs the reference's own output."""
    import os
    dev = _dev()
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_golden_chmult.pt"), weights_only=True)
    c = g["cfg"]
    net = lib.ConditionalUNet(c["in_nc"], c["out_nc"], c["nf"], ch_mult=c["ch_mult"], precision=precision)
    net.load_state_dict(g["state"], strict=True)
    net = net.to(dev)
    tol = 1e-4 if precision == "fp32" else 4e-2 * g["y_int"].abs().max().item()
    assert _maxdiff(net(g["x"].to(dev), g["cond"].to(dev), g["t_int"]), g["y_int"]) < tol
    assert _maxdiff(net(g["x"].to(dev), g["cond"].to(dev), g["t_vec"]), g["y_vec"]) < tol


def test_generate_random_states_bit_exact(lib):
    """Training-time state sampler (sde_utils.py:343-358): the fused kernel == the reference's torch expression, bit for bit,
    also for image sizes that are not a multiple of 4 elements."""
    dev = _dev()
    sde = lib.IRSDE(25, 100, eps=0.005, device=dev)
    for shape in ((4, 3, 16, 20), (3, 3, 9, 7), (1, 1, 5, 5)):
        g = torch.Generator().manual_seed(sum(shape))
        x0, mu = torch.rand(shape, generator=g), torch.rand(shape, generator=g)
        torch.manual_seed(3)
        ts, st = sde.generate_random_states(x0, mu)
        torch.manual_seed(3)
        t2 = torch.randint(1, sde.T + 1, (shape[0], 1, 1, 1)).long()
        noises = torch.randn(shape, device=dev)
        x0d, mud = x0.to(dev), mu.to(dev)
        mean = mud + (x0d - mud) * torch.exp(-sde.thetas_cumsum[t2] * sde.dt)
        ref = noises * sde.sigma_bars[t2] + mean
        assert torch.equal(ts, t2) and torch.equal(st, ref)
