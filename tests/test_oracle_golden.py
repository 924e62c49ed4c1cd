"""Pin the CPU oracle against outputs of the imported reference (tests/golden/make_golden.py)."""
import os
import torch

from oracle import irsde_oracle as O


def _close(a, b, tol):
    d = (a - b).abs().max().item()
    assert d <= tol, d


def test_irsde_schedules(golden):
    for g in golden["irsde_schedules"]:
        ms, T, s, eps = g["args"]
        sc = O.Schedule(ms, T, s, eps)
        for k in ("thetas", "sigmas", "thetas_cumsum", "sigma_bars"):
            assert torch.equal(getattr(sc, k), g[k]), k  # same torch ops => bit-exact
        assert torch.equal(torch.as_tensor(sc.dt), g["dt"])
        assert sc.max_sigma == g["max_sigma"]


def test_schedule_known_answers():
    # SURVEY.md 8(a-1) known answers measured on the reference
    sc = O.Schedule(10, 100, "cosine", 0.005)
    assert abs(float(sc.dt) - 0.10409380) < 1e-7
    assert abs(float(sc.thetas[1]) - 0.00169456) < 1e-7
    assert abs(float(sc.thetas_cumsum[100]) - 50.899448) < 1e-4
    assert abs(float(sc.sigma_bars[100]) - 0.03921520) < 1e-7
    assert abs(float(O.Schedule(10, 50, "cosine", 0.005).dt) - 0.20614207) < 1e-7


def test_dsde_schedules(golden):
    for g in golden["dsde_schedules"]:
        ms, T, s = g["args"]
        sc = O.Schedule(ms, T, s, kind="dsde")
        for k in ("thetas", "sigmas", "thetas_cumsum", "sigma_bars"):
            assert torch.equal(getattr(sc, k), g[k]), k
        for sg, t in g["optimal_t"].items():
            assert O.get_optimal_timestep(sc, sg) == t  # integer work: bit-exact


def test_irsde_steps(golden):
    g = golden["irsde_steps"]
    sc = O.Schedule(*g["args"])
    for st in g["steps"]:
        t, z = st["t"], st["z"]
        assert torch.equal(O.irsde_sde_step(sc, g["x"], g["mu"], g["noise"], z, t), st["sde"])
        assert torch.equal(O.irsde_ode_step(sc, g["x"], g["mu"], g["noise"], t), st["ode"])
        assert torch.equal(O.irsde_posterior_step(sc, g["x"], g["mu"], g["noise"], z, t), st["posterior"])


def test_dsde_steps(golden):
    g = golden["dsde_steps"]
    sc = O.Schedule(*g["args"], kind="dsde")
    for st in g["steps"]:
        assert torch.equal(O.dsde_sde_step(sc, g["x"], g["noise"], st["z"], st["t"]), st["sde"])
        assert torch.equal(O.dsde_ode_step(sc, g["x"], g["noise"], st["t"]), st["ode"])


def test_unet_conditional(golden):
    g = golden["unet_cond"]
    y = O.unet_forward(g["state"], g["xt"], g["cond"], g["t_int"], g["nf"], g["depth"])
    _close(y, g["y_int"], 1e-5)
    y = O.unet_forward(g["state"], g["xt"], g["cond"], g["t_vec"], g["nf"], g["depth"])
    _close(y, g["y_vec"], 1e-5)
    shapes = O.unet_param_shapes(3, 3, g["nf"], g["depth"])
    assert list(shapes) == list(g["state"])  # same names, same registration order
    assert all(tuple(g["state"][k].shape) == tuple(v) for k, v in shapes.items())


def test_unet_denoising_variant(golden):
    g = golden["unet_dsde"]
    y = O.unet_forward(g["state"], g["x"], None, g["t_int"], g["nf"], g["depth"], variant="denoising")
    _close(y, g["y"], 1e-5)
    shapes = O.unet_param_shapes(3, 3, g["nf"], g["depth"], variant="denoising")
    assert list(shapes) == list(g["state"])


def test_chains(golden):
    g = golden["irsde_chain"]
    u = golden["unet_cond"]
    sc = O.Schedule(*g["args"])
    net = lambda x, t: O.unet_forward(u["state"], x, g["lq"], t, u["nf"], u["depth"])
    for mode, c in g["chains"].items():
        x0 = O.reverse_chain(sc, net, g["xT"], g["lq"], c["zs"], mode)
        _close(x0, c["x0"], 2e-4)  # chain is numerically expansive (SURVEY 0); observed ~1e-6
        x5 = O.reverse_chain(sc, net, g["xT"], g["lq"], c["zs"], mode, T=5)
        _close(x5, c["x0_T5"], 2e-4)


def test_dsde_chain(golden):
    g = golden["unet_dsde"]
    sc = O.Schedule(*g["args"], kind="dsde")
    net = lambda x, t: O.unet_forward(g["state"], x, None, t, g["nf"], g["depth"], variant="denoising")
    assert O.get_optimal_timestep(sc, 25) == g["Tstar"]
    _close(O.reverse_chain(sc, net, g["x"], None, g["zs"], "dsde_sde", T=g["Tstar"]), g["x0_sde"], 2e-4)
    _close(O.reverse_chain(sc, net, g["x"], None, g["zs"], "dsde_ode", T=g["Tstar"]), g["x0_ode"], 2e-4)


def test_nafnet_oracle_vs_reference():
    import os
    g_all = torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_golden_nafnet.pt"), weights_only=True)
    for key, g in g_all.items():
        c = g["cfg"]
        args = (c["width"], c["enc_blk_nums"], c["middle_blk_num"], c["dec_blk_nums"])
        y = O.nafnet_forward(g["state"], g["x"], g["cond"], g["t_int"], *args, latent=g["latent"])
        _close(y, g["y"], 1e-5)
        yv = O.nafnet_forward(g["state"], g["x"], g["cond"], g["t_vec"], *args, latent=g["latent"])
        _close(yv, g["y_vec"], 1e-5)
        shapes = O.nafnet_param_shapes(c["img_channel"], c["width"], c["middle_blk_num"], c["enc_blk_nums"], c["dec_blk_nums"])
        assert list(shapes) == list(g["state"])


def test_latent_unet_oracle_vs_reference():
    import os
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_golden_latent.pt"), weights_only=True)
    c = g["cfg"]
    z, h = O.latent_unet_encode(g["state"], g["x"], c["ch_mult"])
    _close(z, g["z"], 1e-5)
    y = O.latent_unet_decode(g["state"], g["z2"], h, c["ch_mult"], g["x"].shape[2], g["x"].shape[3])
    _close(y, g["y"], 1e-5)
    shapes = O.latent_unet_param_shapes(c["in_ch"], c["out_ch"], c["ch"], c["ch_mult"], c["embed_dim"])
    assert list(shapes) == list(g["state"])


def test_latent_unet_oracle_real_checkpoint():
    """The shipped latent-dehazing.pth (2.0 M params) through the reference module vs the oracle (staged under oracle/_ref by build())."""
    import os
    import sys
    ref = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
    ck = os.path.join(ref, "codes", "config", "latent-dehazing", "pretrained_models", "latent-dehazing.pth")
    if not os.path.exists(ck):
        import pytest
        pytest.skip("oracle/_ref not staged")
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    from make_golden_latent import load_unet_arch
    arch = load_unet_arch()
    sd = torch.load(ck, map_location="cpu", weights_only=True)
    net = arch.UNet(in_ch=3, out_ch=3, ch=8, ch_mult=[4, 8, 8, 16], embed_dim=8).eval()
    net.load_state_dict(sd, strict=True)
    x = torch.rand(1, 3, 50, 70, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        z, h = net.encode(x)
        y = net.decode(z, h)
    zo, ho = O.latent_unet_encode(sd, x, [4, 8, 8, 16])
    _close(zo, z, 1e-4)
    for a, b in zip(ho, h):
        _close(a, b, 1e-3)
    # decode is NOT compared for this checkpoint: on such inputs the reference's own fp32 and fp64 decodes differ by
    # O(100) (ill-conditioned trained weights), so no fp32 restatement can be pinned there; decode parity is pinned on
    # the well-conditioned random-weight fixture (test_latent_unet_oracle_vs_reference).
    assert y.shape == x.shape
    assert list(O.latent_unet_param_shapes(3, 3, 8, [4, 8, 8, 16], 8)) == list(sd)
    # A natural image (images/1.png crop): the oracle follows the reference's fp32 op order closely enough to reproduce
    # its decode to 1e-5 of the output range, although that range is ~78 and the reference's fp32 and fp64 runs differ by
    # 0.17 in z and ~67 in y here - the checkpoint is ill-conditioned, so this pins the restatement, not a tolerance a
    # re-ordered fp32 implementation (the GPU kernels) can be held to.
    import cv2
    import numpy as np
    img = cv2.imread(os.path.join(ref, "images", "1.png"))
    xi = torch.from_numpy(img[:, :, [2, 1, 0]].astype(np.float32) / 255.).permute(2, 0, 1)[None][:, :, :160, :224].contiguous()
    with torch.no_grad():
        zi, hi = net.encode(xi)
        yi = net.decode(zi, hi)
    zo, ho = O.latent_unet_encode(sd, xi, [4, 8, 8, 16])
    yo = O.latent_unet_decode(sd, zo, ho, [4, 8, 8, 16], 160, 224)
    _close(zo, zi, 1e-4)
    assert (yo - yi).abs().max().item() < 1e-4 * yi.abs().max().item()


# ---- image helpers (oracle/imaging_oracle.py vs the reference's img_utils outputs) ---------------------------
def _imaging_golden():
    import os
    import numpy as np
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_golden_imaging.npz"))


def test_imaging_oracle_matches_reference():
    import numpy as np
    from oracle import imaging_oracle as IO
    g = _imaging_golden()
    for k in "abc":
        t = g["t_" + k]
        t2 = t[0] if t.shape[0] == 1 else t
        assert np.array_equal(IO.tensor2img(t2), g["img_" + k])                              # bit exact, incl. .5 ties
        assert np.array_equal(IO.tensor2img(t2 * np.float32(2) - np.float32(1), (-1, 1)), g["img11_" + k])
    assert np.array_equal(IO.img2tensor(g["x"]), g["x_tensor"])
    assert IO.calculate_psnr(g["x"], g["y"]) == float(g["psnr"])                            # exact integer sums
    assert IO.calculate_psnr(g["x"][4:-4, 4:-4], g["y"][4:-4, 4:-4]) == float(g["psnr_crop4"])
    assert IO.calculate_psnr(g["x"], g["x"]) == float("inf")
    assert abs(IO.calculate_ssim(g["x"], g["y"]) - float(g["ssim"])) < 1e-12
    assert abs(IO.calculate_ssim(g["x"][4:-4, 4:-4], g["y"][4:-4, 4:-4]) - float(g["ssim_crop4"])) < 1e-12
    assert abs(IO.calculate_ssim(g["x"][:, :, 0], g["y"][:, :, 0]) - float(g["ssim_gray"])) < 1e-12


def test_unet_ch_mult_variant_vs_reference():
    """ConditionalUNet(in_nc, out_nc, nf, ch_mult=[...]) of the latent tasks (latent-dehazing/.../DenoisingUNet_arch.py:20):
    oracle and state-dict table against the reference's own output."""
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_golden_chmult.pt"), weights_only=True)
    c = g["cfg"]
    shapes = O.unet_param_shapes(c["in_nc"], c["out_nc"], c["nf"], c["ch_mult"])
    assert list(shapes.keys()) == list(g["state"].keys())
    assert all(tuple(g["state"][k].shape) == tuple(v) for k, v in shapes.items())
    y = O.unet_forward(g["state"], g["x"], g["cond"], g["t_int"], c["nf"], c["ch_mult"])
    assert (y - g["y_int"]).abs().max().item() < 1e-5
    y = O.unet_forward(g["state"], g["x"], g["cond"], g["t_vec"], c["nf"], c["ch_mult"])
    assert (y - g["y_vec"]).abs().max().item() < 1e-5
    import irsde_b200
    m = irsde_b200.ConditionalUNet(c["in_nc"], c["out_nc"], c["nf"], ch_mult=c["ch_mult"])
    assert list(m.state_dict().keys()) == list(g["state"].keys())
    m.load_state_dict(g["state"], strict=True)
    m2 = irsde_b200.ConditionalUNet(c["in_nc"], c["out_nc"], c["nf"], c["ch_mult"])   # positional, like the reference signature
    assert m2.depth == 3 and list(m2.state_dict().keys()) == list(g["state"].keys())


def test_oracle_per_layer_trace_vs_reference_hooks():
    """The oracle's `trace=` checkpoints (what the GPU per-layer parity reports compare with) against forward hooks on the
    reference's own modules (tests/golden/make_golden_layers.py): every layer's fingerprint - shape, fp64 sum / abs-sum,
    <= 512 strided elements - for the conditional UNet (ragged input) and the denoising-sde variant (full Attention)."""
    import _golden
    G = _golden.load("reference_golden_layers.pt")
    for variant, g in (("conditional", G["cond"]), ("denoising", G["denoising"])):
        c = g["cfg"]
        tr = {}
        y = O.unet_forward(g["state"], g["x"], g.get("cond"), g["t"], c["nf"], c["depth"], variant=variant, trace=tr)
        assert (y - g["y"]).abs().max().item() < 1e-5
        assert set(tr.keys()) == set(g["layers"].keys()), (sorted(set(tr) ^ set(g["layers"])))
        for key, fp in g["layers"].items():
            t = tr[key]
            assert list(t.shape) == fp["shape"].tolist(), key
            f = t.reshape(-1)
            n = f.numel()
            scale = max(1.0, float(fp["abssum"]) / n)
            assert (f[::int(fp["stride"])] - fp["sample"]).abs().max().item() < 1e-5 * max(1.0, float(fp["sample"].abs().max())), key
            assert abs(float(f.double().sum()) - float(fp["sum"])) < 2e-6 * n * scale, key
            assert abs(float(f.double().abs().sum()) - float(fp["abssum"])) < 2e-6 * n * scale, key
