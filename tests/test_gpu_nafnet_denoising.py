"""The denoising-sde task's ConditionalNAFNet (irsde_b200.DenoisingNAFNet: no condition, intro over img_channel channels)
driven by DenoisingSDE on the native library: forward and chains against the reference's own outputs
(tests/golden/make_golden_nafnet_dsde.py), bit-identical execution paths, the refusion.yml size, and the pairings the
library refuses."""
import os

import pytest
import torch

import _nafnet_denoising_oracle as D

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "reference_golden_nafnet_dsde.pt"), weights_only=True)


def _maxdiff(a, b):
    return (a.detach().float().cpu() - b.float().cpu()).abs().max().item()


def _net(lib, state, cfg, precision, dev, force_simt=False):
    net = lib.DenoisingNAFNet(precision=precision, force_simt=force_simt, **cfg)
    net.load_state_dict(state, strict=True)
    return net.to(dev)


@pytest.mark.parametrize("precision,force_simt", [("fp32", False), ("fp32x3", False), ("bf16", False), ("bf16", True)])
def test_forward_vs_reference(gold, precision, force_simt):
    """Zero pad 18x23 -> 20x24, scalar and per-image t.  fp32 / fp32x3 within 1e-4; bf16 within 4 % of max|y|."""
    import irsde_b200 as lib
    dev = _dev()
    net = _net(lib, gold["state"], gold["cfg"], precision, dev, force_simt)
    x = gold["x"].to(dev)
    for t, ref in ((gold["t_int"], gold["y"]), (gold["t_vec"], gold["y_vec"])):
        y = net(x, t)
        assert y.shape == ref.shape
        tol = 1e-4 if precision != "bf16" else 4e-2 * ref.abs().max().item()
        assert _maxdiff(y, ref) < tol, (precision, force_simt, _maxdiff(y, ref))
    assert net.launch_count() > 0


@pytest.mark.parametrize("precision", ["fp32", "fp32x3"])
@pytest.mark.parametrize("graph", [True, False])
def test_dsde_chains_vs_reference(gold, precision, graph):
    """reverse_sde (pre-drawn z) and reverse_ode from T* = get_optimal_timestep(25), with T the 0-dim LongTensor that
    denoising_model.py:163 passes: within 1e-3 of the reference's own chains."""
    import irsde_b200 as lib
    dev = _dev()
    net = _net(lib, gold["state"], gold["cfg"], precision, dev)
    sde = lib.DenoisingSDE(*gold["args"], device=dev)
    sde.use_graph = graph
    sde.set_model(net)
    T = sde.get_optimal_timestep(gold["sigma"])
    assert torch.is_tensor(T) and T.dim() == 0 and int(T) == gold["Tstar"] == 22
    xn = gold["xn"].to(dev)
    assert _maxdiff(sde.reverse_sde(xn, T=T, zs=gold["zs"].to(dev)), gold["x0_sde"]) < 1e-3
    assert _maxdiff(sde.reverse_ode(xn, T=T), gold["x0_ode"]) < 1e-3


def _small(lib, precision, dev):
    cfg = dict(img_channel=3, width=16, middle_blk_num=1, enc_blk_nums=[1, 1], dec_blk_nums=[1, 1])
    P = D.make_weights(3, 16, 1, [1, 1], [1, 1], seed=4)
    net = _net(lib, P, cfg, precision, dev)
    sde = lib.DenoisingSDE(70, 100, device=dev)
    sde.set_model(net)
    g = torch.Generator().manual_seed(11)
    x = torch.rand(3, 3, 34, 42, generator=g)                  # pads to 36 x 44
    xn = (x + torch.randn(x.shape, generator=g) * 0.1).to(dev)
    zs = torch.randn((12,) + tuple(x.shape), generator=g).to(dev)
    return net, sde, xn, zs


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_stepwise_loop_equals_library_chain(precision):
    """noise_fn + the step kernel per step (the path save_states=True takes) == the captured chain, bit for bit."""
    import irsde_b200 as lib
    dev = _dev()
    net, sde, xn, zs = _small(lib, precision, dev)
    T = 12
    for mode, name in ((lib._lib.MODE_DSDE_SDE, "reverse_sde"), (lib._lib.MODE_DSDE_ODE, "reverse_ode")):
        a = getattr(sde, name)(xn, T=T, zs=zs)
        x = xn.clone()
        for i, t in enumerate(reversed(range(1, T + 1))):
            x = sde._native_step(mode, x, None, net(x, t), zs[i] if mode == lib._lib.MODE_DSDE_SDE else None, t)
        assert torch.equal(a, x), (name, (a - x).abs().max().item())


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_graph_replay_equals_eager(precision):
    import irsde_b200 as lib
    dev = _dev()
    _, sde, xn, zs = _small(lib, precision, dev)
    out = {}
    for graph in (True, False):
        sde.use_graph = graph
        out[graph] = (sde.reverse_sde(xn, T=12, zs=zs), sde.reverse_ode(xn, T=12))
    assert torch.equal(out[True][0], out[False][0]) and torch.equal(out[True][1], out[False][1])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_image_in_batch_equals_image_alone(precision):
    """With the in-kernel Philox keyed per image, image 1 of a batch of 3 == the same image run alone as uid 1."""
    import irsde_b200 as lib
    dev = _dev()
    _, sde, xn, _ = _small(lib, precision, dev)
    sde.rng, sde.seed, sde.seed_auto_increment = "philox", 17, False
    full = sde.reverse_sde(xn, T=12)
    sde.image_base = 1
    one = sde.reverse_sde(xn[1:2].contiguous(), T=12)
    assert torch.equal(full[1:2], one)
    sde.image_base = 0                                          # the same image as uid 0 draws other noise
    assert not torch.equal(one, sde.reverse_sde(xn[1:2].contiguous(), T=12))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_chain_on_non_blocking_stream_equals_default_stream(precision):
    import irsde_b200 as lib
    dev = _dev()
    _, sde, xn, zs = _small(lib, precision, dev)
    a = (sde.reverse_sde(xn, T=12, zs=zs), sde.reverse_ode(xn, T=12))
    s = torch.cuda.Stream(device=dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        b = (sde.reverse_sde(xn, T=12, zs=zs), sde.reverse_ode(xn, T=12))
    torch.cuda.current_stream(dev).wait_stream(s)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_refusion_yml_size_bf16():
    """options/test/refusion.yml: width 64, enc [1,1,1,28], middle 1, dec [1,1,1,1], DenoisingSDE(70, 1000) at Kodak size
    1x3x512x768.  A few ODE steps: finite, and graph replay == eager launch bit for bit."""
    import irsde_b200 as lib
    dev = _dev()
    torch.manual_seed(0)
    net = lib.DenoisingNAFNet(3, 64, 1, [1, 1, 1, 28], [1, 1, 1, 1], precision="bf16")
    with torch.no_grad():
        for n, p in net.named_parameters():
            if n.endswith("beta") or n.endswith("gamma"):
                p.fill_(0.1)      # the reference initialises them to zero: every block would be the identity
    net = net.to(dev)
    sde = lib.DenoisingSDE(70, 1000, device=dev)
    sde.set_model(net)
    assert int(sde.get_optimal_timestep(15)) == 158
    g = torch.Generator().manual_seed(2)
    xn = torch.rand(1, 3, 512, 768, generator=g).to(dev)
    out = {}
    for graph in (True, False):
        sde.use_graph = graph
        out[graph] = sde.reverse_ode(xn, T=3)
    assert torch.isfinite(out[True]).all()
    assert torch.equal(out[True], out[False])
    assert not torch.equal(out[True], xn)


def test_refused_pairings():
    import irsde_b200 as lib
    from irsde_b200 import nafnet
    dev = _dev()
    g = torch.Generator().manual_seed(1)
    x = torch.rand(1, 3, 16, 16, generator=g).to(dev)
    dn = lib.DenoisingNAFNet(3, 8, 1, [1], [1]).to(dev)
    irsde = lib.IRSDE(10, 5, device=dev)
    irsde.set_model(dn)
    irsde.set_mu(x)
    for name in ("reverse_sde", "reverse_ode", "reverse_posterior"):       # IRSDE modes on the denoising NAFNet
        with pytest.raises(lib._lib.IrsdeError, match="variant"):
            getattr(irsde, name)(x)
    cn = lib.ConditionalNAFNet(3, 8, 1, [1], [1]).to(dev)
    dsde = lib.DenoisingSDE(70, 100, device=dev)
    dsde.set_model(cn)
    for name in ("reverse_sde", "reverse_ode"):                              # DSDE modes on the conditional NAFNet
        with pytest.raises(lib._lib.IrsdeError, match="variant"):
            getattr(dsde, name)(x, T=5)
    with pytest.raises(lib._lib.IrsdeError, match="mu required"):          # the conditional NAFNet still needs mu
        cn._run(x, None, 3)
    with pytest.raises(lib._lib.IrsdeError, match="latent"):
        nafnet._NafContext(3, 8, 1, [1], [1], True, lib._lib.PREC_FP32, 0, variant=lib._lib.NET_DENOISING)
    with pytest.raises(lib._lib.IrsdeError, match="bad variant"):
        nafnet._NafContext(3, 8, 1, [1], [1], False, lib._lib.PREC_FP32, 0, variant=2)
