"""Every network the benchmark workloads run, at its real architecture, batch and image size, against the oracle run in
float64 on the GPU, in all three precisions:

- c2 / c3: ConditionalUNet nf=64 depth=4 on 8x3x256x256 at t = 100, 50, 1 and with a different t per image;
- c5: the same network on 2x3x512x512 at t = 400, 200, 1;
- c4 encode / decode: the latent UNet(3, 3, 64, [1, 2, 4], 4) on 1x3x1024x1024.  Encode is compared with the 4x256x256
  latent; decode takes the oracle's latent and the skips the GPU's own encode left behind.  This runs the fused
  LinearAttention block at C = 128 on 256x256 and the unfused one at C = 256;
- c4 score network: the latent ConditionalNAFNet w=64 enc [1, 1, 1, 28] dec [1, 1, 1, 1] on 16 latent tiles of 128x128
  at t = 200, 100, 1.

The network input is the x_t of the workload's own schedule, and each sampler step of the workload (reverse_sde for c2
and c4, reverse_posterior for c5) is checked teacher-forced: `_native_step` fed the fp64 oracle's noise estimate (as fp32)
and the same z, against the oracle's step in float64.

Bounds, relative to the output's scale:
- fp32 and fp32x3: max|err| / max|ref|, the accuracy class of the 1e-4-per-forward tests;
- bf16 keeps two global bounds (max|err| / max|ref| and RMS(err) / RMS(ref)) and adds a spatial one.  The error is cut
  into (image, 32x32 block) cells, each cell's statistic is RMS(err in the cell) / RMS(ref over the whole output), and the
  largest cell must stay within CELL_RATIO times the median cell.  A wiring error of the launch plan that touches one skip,
  one image's time row, or one tile or border of a conv launch leaves the global bounds nearly unchanged but puts a few
  cells far above the rest.
Before any output is accepted, every case shows that its bounds reject wrong references: the batch rolled by one image,
the oracle at t - 1 and at t + 1, one 32x32 block of one image shifted by a pixel and, for the score network, one tile's
reference taken from its neighbour.

Measured on an H100 80GB HBM3 at 700 W (the largest over the calls of a case; max = max|err| / max|ref|, rms = RMS(err) / RMS(ref),
cell = largest / median cell; peak = the largest over the three precisions; wall = fp64 oracle + the three precisions):

  case        fp32 max  fp32x3 max  bf16 max  bf16 rms  bf16 cell  peak    wall
  c2          7.5e-6    6.7e-6      2.3e-2    1.15e-2   1.24       8.2 GB  4.9 + 10.4 s
  c5          6.7e-6    6.8e-6      1.9e-2    1.13e-2   1.12       8.3 GB  4.0 + 9.8 s
  c4 encode   2.0e-6    1.6e-6      1.0e-2    7.6e-3    1.02       6.7 GB  0.3 + 0.6 s (with decode)
  c4 decode   2.0e-6    1.8e-6      1.1e-2    1.11e-2   1.06
  c4 NAFNet   1.2e-5    1.4e-5      2.9e-2    2.85e-2   1.08       3.5 GB  1.1 + 5.7 s

The teacher-forced steps come to 0.25 of their bound.  Every wrong reference lands at least 5x past the bf16 bounds and
thousands of times past the fp32 ones.  Two deliberate breaks of the bf16 plan were tried on c2 and both fail the test:
writing the skip of downs.1 8 channels off (every call, RMS 0.37-0.41 of the output) and handing image 3 the time row of
image 4 (the per-image call: max 0.25, largest cell 19.7x the median).  The autoencoder runs one image, so its wrong reference is the shifted block alone.

Every case states a device-memory budget (at most 24 GB) in its id and skips when that much is not free; it prints its
peak (torch's reserved peak plus the library's device bytes), its errors and its runtime.

The last test runs the c2 bf16 forward, a 3-step graph chain and the c4 NAFNet forward in two processes, one with
IRSDE_PDL=1 and one with IRSDE_PDL=0 (the library reads the switch once per process), and requires bit-identical results.
"""
import contextlib
import math
import os
import subprocess
import sys
import time

import pytest
import torch
from torch.overrides import TorchFunctionMode

from oracle import irsde_oracle as O

GB = 1 << 30
BUDGET = 24 * GB
CELL = 32
U = 2.0 ** -24

# bounds: the measured values of the module docstring with a margin of 1.4x to 3x
MAX_FP32 = {"c2": 2e-5, "c5": 2e-5, "c4-encode": 1e-5, "c4-decode": 1e-5, "c4-nafnet": 3e-5}
MAX_BF16 = {"c2": 3.5e-2, "c5": 3e-2, "c4-encode": 1.5e-2, "c4-decode": 1.6e-2, "c4-nafnet": 4.5e-2}
RMS_BF16 = {"c2": 1.6e-2, "c5": 1.6e-2, "c4-encode": 1.1e-2, "c4-decode": 1.6e-2, "c4-nafnet": 4e-2}
CELL_RATIO = {"c2": 2.0, "c5": 2.0, "c4-encode": 2.0, "c4-decode": 2.0, "c4-nafnet": 2.0}
STEP_BOUND = 4.0   # step error within 4x max(what fp32 torch gets on the same step, 2^-24 max|ref|)


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def _gb(n):
    return "%.1f GB" % (n / GB)


# ------------------------------------------------------------------------------------------------------------------
# the oracle in float64 on a device
# ------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _fp64_on(device):
    """Tensors the oracle creates itself (torch.tensor([t]), the arange of the time embeddings) are created on `device`
    and, when floating point, in float64."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        with torch.device(device):
            yield
    finally:
        torch.set_default_dtype(old)


def _to64(P, device):
    return {k: v.to(device, torch.float64) for k, v in P.items()}


def _times64(ts, device):
    """Integer time steps as an int64 tensor: the oracle casts a floating-point time to fp32 before its time embedding and
    leaves an integer one alone, so the embedding is computed in float64."""
    return torch.tensor([int(t) for t in ts], dtype=torch.int64, device=device)


def _oracle64(fn, P64, *args, device, **kw):
    """fn(P64, *args, **kw) in float64 on `device`; tensor arguments are moved there, floating-point ones as float64."""
    args = [a.to(device, torch.float64) if torch.is_tensor(a) and a.is_floating_point() else a for a in args]
    with _fp64_on(device), torch.no_grad():
        return fn(P64, *args, **kw)


class _DtypeAudit(TorchFunctionMode):
    """Records the (dtype, device type) of every floating-point tensor a torch call returns."""

    def __init__(self):
        super().__init__()
        self.seen = set()

    def __torch_function__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        for o in (out if isinstance(out, (tuple, list)) else (out,)):
            if torch.is_tensor(o) and o.is_floating_point():
                self.seen.add((o.dtype, o.device.type))
        return out


def test_fp64_oracle_wrapper_matches_fp32_oracle_on_cpu():
    """The wrapped oracle on a small config of each network, on the CPU: within fp32 rounding of the plain fp32 oracle
    (and not equal to it, so it did not run in fp32), with every traced activation and every floating-point tensor any
    torch call returned in float64."""
    cpu = torch.device("cpu")
    g = torch.Generator().manual_seed(0)
    x = torch.rand(2, 3, 18, 22, generator=g)
    cond = torch.rand(2, 3, 18, 22, generator=g)
    ts = [7, 60]
    results = []

    P = O.make_weights(3, 3, 8, 2, seed=3)
    trace = {}
    audit = _DtypeAudit()
    with audit:
        y64 = _oracle64(O.unet_forward, _to64(P, cpu), x, cond, _times64(ts, cpu), 8, 2, trace=trace, device=cpu)
    assert len(trace) > 20 and all(v.dtype == torch.float64 for v in trace.values()), \
        sorted(k for k, v in trace.items() if v.dtype != torch.float64)
    results.append(("unet", audit.seen, y64, O.unet_forward(P, x, cond, torch.tensor(ts), 8, 2)))

    Pn = O.make_nafnet_weights(4, 16, 1, [1, 1], [1, 1], seed=4)
    xn, cn = torch.rand(2, 4, 12, 20, generator=g), torch.rand(2, 4, 12, 20, generator=g)
    audit = _DtypeAudit()
    with audit:
        y64 = _oracle64(O.nafnet_forward, _to64(Pn, cpu), xn, cn, _times64(ts, cpu), 16, [1, 1], 1, [1, 1], latent=True,
                        device=cpu)
    results.append(("nafnet", audit.seen, y64, O.nafnet_forward(Pn, xn, cn, torch.tensor(ts), 16, [1, 1], 1, [1, 1], latent=True)))

    Pa = O.make_latent_unet_weights(3, 3, 8, [1, 2], 4, seed=5)
    audit = _DtypeAudit()
    with audit:
        z64, h64 = _oracle64(O.latent_unet_encode, _to64(Pa, cpu), x, [1, 2], device=cpu)
        d64 = _oracle64(O.latent_unet_decode, _to64(Pa, cpu), z64, h64, [1, 2], 18, 22, device=cpu)
    z32, h32 = O.latent_unet_encode(Pa, x, [1, 2])
    results.append(("latent encode", audit.seen, z64, z32))
    results.append(("latent decode", audit.seen, d64, O.latent_unet_decode(Pa, z32, h32, [1, 2], 18, 22)))
    assert all(h.dtype == torch.float64 for h in h64)

    for name, seen, y64, y32 in results:
        assert seen == {(torch.float64, "cpu")}, (name, seen)
        assert y64.dtype == torch.float64 and y64.shape == y32.shape, name
        d = (y64 - y32.double()).abs().max().item()
        scale = y32.abs().max().item()
        assert 0 < d <= 1e-5 * scale, (name, d, scale)


# ------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------
def _case(key, name, need_gb, **kw):
    c = dict(key=key, name=name, need=int(need_gb * GB), **kw)
    assert c["need"] <= BUDGET
    c["id"] = "%s, %s" % (name, _gb(c["need"]))
    return c


CASES = [
    _case("c2", "c2/c3 ConditionalUNet nf64 d4 8x3x256x256", 12, net="unet", B=8, H=256, W=256, T=100, max_sigma=10,
          mode="sde", ts=[100, 50, 1], mixed=[100, 50, 1, 73, 2, 99, 51, 10], tpm=50, seed=0),
    _case("c5", "c5 ConditionalUNet nf64 d4 2x3x512x512", 12, net="unet", B=2, H=512, W=512, T=400, max_sigma=10,
          mode="posterior", ts=[400, 200, 1], mixed=None, tpm=200, seed=0),
    _case("c4-ae", "c4 latent UNet(3,3,64,[1,2,4],4) encode/decode 1x3x1024x1024", 10, net="latent", B=1, H=1024, W=1024,
          seed=2),
    _case("c4-nafnet", "c4 latent NAFNet w64 [1,1,1,28] on 16 tiles of 4x128x128", 6, net="nafnet", B=16, H=128, W=128,
          T=200, max_sigma=50, mode="sde", ts=[200, 100, 1], mixed=None, tpm=100, seed=6),
]
PRECISIONS = ["fp32", "fp32x3", "bf16"]
NAF = dict(img_channel=4, width=64, middle_blk_num=1, enc_blk_nums=[1, 1, 1, 28], dec_blk_nums=[1, 1, 1, 1])
AE = dict(in_ch=3, out_ch=3, ch=64, ch_mult=[1, 2, 4], embed_dim=4)


def _weights(c):
    if c["net"] == "unet":
        return O.make_weights(3, 3, 64, 4, seed=c["seed"])
    if c["net"] == "nafnet":
        return O.make_nafnet_weights(4, 64, 1, NAF["enc_blk_nums"], NAF["dec_blk_nums"], seed=c["seed"])
    return O.make_latent_unet_weights(3, 3, 64, AE["ch_mult"], 4, seed=c["seed"])


def _schedule(c):
    return O.Schedule(c["max_sigma"], c["T"], "cosine", 0.005)


def _x_t(sc, mu, x0, n, ts):
    """x_t = mu + (x0 - mu) exp(-thetā_t dt) + sigmā_t n (float64), one t per image."""
    m = torch.tensor([math.exp(-float(sc.thetas_cumsum[t]) * float(sc.dt)) for t in ts], dtype=torch.float64)
    sb = torch.tensor([float(sc.sigma_bars[t]) for t in ts], dtype=torch.float64)
    return mu + (x0 - mu) * m[:, None, None, None] + sb[:, None, None, None] * n


def _inputs(c, dev):
    """fp32 inputs (the network sees exactly these; the oracle gets them as float64).  Calls: [(label, ts, x_t)]."""
    g = torch.Generator().manual_seed(100 + c["seed"])
    B, H, W = c["B"], c["H"], c["W"]
    if c["net"] == "latent":
        return dict(x=torch.rand(B, 3, H, W, generator=g).to(dev))
    ch = 4 if c["net"] == "nafnet" else 3
    shape = (B, ch, H, W)
    mu, x0 = torch.rand(shape, generator=g, dtype=torch.float64), torch.rand(shape, generator=g, dtype=torch.float64)
    n, z = torch.randn(shape, generator=g, dtype=torch.float64), torch.randn(shape, generator=g, dtype=torch.float64)
    sc = _schedule(c)
    calls = [("t=%d" % t, [t] * B, _x_t(sc, mu, x0, n, [t] * B).float().to(dev)) for t in c["ts"]]
    if c["mixed"]:
        calls.append(("t per image %s" % c["mixed"], list(c["mixed"]), _x_t(sc, mu, x0, n, c["mixed"]).float().to(dev)))
    return dict(mu=mu.float().to(dev), z=z.float().to(dev), calls=calls, sc=sc)


_REFS = {}


def _oracle_refs(c, dev):
    """The oracle's outputs of a case (computed once, shared by the three precisions), with its own peak and time."""
    if c["key"] in _REFS:
        return _REFS[c["key"]]
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    inp = _inputs(c, dev)
    P64 = _to64(_weights(c), dev)
    refs = dict(inp=inp)
    if c["net"] == "latent":
        z, h = _oracle64(O.latent_unet_encode, P64, inp["x"], AE["ch_mult"], device=dev)
        refs["encode"] = z
        refs["decode"] = _oracle64(O.latent_unet_decode, P64, z, h, AE["ch_mult"], c["H"], c["W"], device=dev)
        del h
    else:
        if c["net"] == "unet":
            fwd = lambda x, ts: _oracle64(O.unet_forward, P64, x, inp["mu"], _times64(ts, dev), 64, 4, device=dev)
        else:
            fwd = lambda x, ts: _oracle64(O.nafnet_forward, P64, x, inp["mu"], _times64(ts, dev), 64, NAF["enc_blk_nums"],
                                          1, NAF["dec_blk_nums"], latent=True, device=dev)
        refs["calls"] = [fwd(x, ts) for _, ts, x in inp["calls"]]
        k = c["ts"].index(c["tpm"])
        x = inp["calls"][k][2]
        refs["t-1"] = fwd(x, [c["tpm"] - 1] * c["B"])
        refs["t+1"] = fwd(x, [c["tpm"] + 1] * c["B"])
    torch.cuda.synchronize()
    del P64
    refs["peak"] = torch.cuda.max_memory_reserved()
    refs["seconds"] = time.perf_counter() - t0
    torch.cuda.empty_cache()
    _REFS.clear()   # one case's references at a time
    _REFS[c["key"]] = refs
    return refs


# ------------------------------------------------------------------------------------------------------------------
# error statistics and bounds
# ------------------------------------------------------------------------------------------------------------------
def _cells(err, ref):
    """RMS(err) in each (image, 32x32 block) cell over all channels, divided by RMS(ref) over the whole output."""
    B, C, H, W = err.shape
    assert H % CELL == 0 and W % CELL == 0
    e = err.double().pow(2).reshape(B, C, H // CELL, CELL, W // CELL, CELL).mean(dim=(1, 3, 5)).sqrt()
    return e / ref.double().pow(2).mean().sqrt()


def _stats(got, ref):
    d = got.double() - ref
    cells = _cells(d, ref)
    med = cells.median().item()
    return dict(max=d.abs().max().item() / ref.abs().max().item(),
                rms=(d.pow(2).mean() / ref.pow(2).mean()).sqrt().item(),
                cell=cells.max().item() / med if med > 0 else math.inf)


def _ratio(key, prec, s):
    """Largest statistic / its bound: <= 1 passes."""
    if prec != "bf16":
        return s["max"] / MAX_FP32[key]
    return max(s["max"] / MAX_BF16[key], s["rms"] / RMS_BF16[key], s["cell"] / CELL_RATIO[key])


def _shift_block(ref, b, by, bx):
    """ref with the 32x32 block (by, bx) of image b read one pixel further down."""
    r = ref.clone()
    y0, x0 = by * CELL, bx * CELL
    r[b, :, y0:y0 + CELL, x0:x0 + CELL] = ref[b, :, y0 + 1:y0 + CELL + 1, x0:x0 + CELL]
    return r


def _wrong_refs(c, ref, refs=None):
    """[(label, wrong reference)] for the call at t = tpm (or the single output of the autoencoder)."""
    B, H, W = ref.shape[0], ref.shape[2], ref.shape[3]
    out = [("one block shifted by a pixel", _shift_block(ref, B - 1, H // CELL // 2, W // CELL // 2 - 1))]
    if B > 1:
        out.append(("batch rolled by one image", torch.roll(ref, 1, dims=0)))
    if refs is not None:
        out += [("oracle at t-1", refs["t-1"]), ("oracle at t+1", refs["t+1"])]
    if c["net"] == "nafnet":
        r = ref.clone()
        r[5] = ref[6]
        out.append(("tile 5 from its neighbour", r))
    return out


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import irsde_b200
    return irsde_b200


@pytest.fixture
def budget(request):
    """Skips unless the case's bytes are free, and frees everything the case allocated afterwards."""
    c = request.node.callspec.params["case"]
    _dev()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < c["need"]:
        pytest.skip("needs %d bytes of device memory, %d free" % (c["need"], free))
    yield c
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _net(lib, c, prec, P, dev):
    if c["net"] == "unet":
        net = lib.ConditionalUNet(3, 3, 64, depth=4, precision=prec)
    elif c["net"] == "nafnet":
        net = lib.ConditionalNAFNet(latent=True, precision=prec, **NAF)
    else:
        net = lib.UNet(precision=prec, **AE)
    net.load_state_dict(P, strict=True)
    return net.to(dev)


def _step_check(lib, c, net, inp, refs, dev):
    """Teacher-forced sampler steps at each t of the case: [(t, ratio to the bound, [(wrong label, ratio)])]."""
    sde = lib.IRSDE(c["max_sigma"], c["T"], schedule="cosine", eps=0.005, device=dev)
    sde.set_model(net)
    sc = inp["sc"]
    mode = {"sde": lib._lib.MODE_SDE, "posterior": lib._lib.MODE_POSTERIOR}[c["mode"]]
    fn = {"sde": O.irsde_sde_step, "posterior": O.irsde_posterior_step}[c["mode"]]
    mu, z = inp["mu"], inp["z"]
    rows = []
    for k, t in enumerate(c["ts"]):
        x = inp["calls"][k][2]
        eps = refs["calls"][k].float()
        got = sde._native_step(mode, x, mu, eps, z, t).double()
        ref = fn(sc, x.double(), mu.double(), eps.double(), z.double(), t)
        err32 = (fn(sc, x, mu, eps, z, t).double() - ref).abs().max().item()
        lim = STEP_BOUND * max(err32, U * ref.abs().max().item())
        r = lambda a: (got - a).abs().max().item() / lim
        t2 = t + 1 if t == 1 else t - 1
        wrong = [("t=%d coefficients" % t2, r(fn(sc, x.double(), mu.double(), eps.double(), z.double(), t2)))]
        # the posterior's std at t = 1 is sqrt(1e-20 dt) * max_sigma: z has no effect there
        if c["B"] > 1 and not (c["mode"] == "posterior" and t == 1):
            wrong.append(("z rolled by one image", r(fn(sc, x.double(), mu.double(), eps.double(), torch.roll(z, 1, 0).double(), t))))
        rows.append((t, r(ref), wrong))
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_workload_network_vs_fp64_oracle(lib, case, prec, budget, capsys):
    c = case
    dev = _dev()
    refs = _oracle_refs(c, dev)
    inp = refs["inp"]
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    net = _net(lib, c, prec, _weights(c), dev)
    results, wrong, steps = [], [], []
    if c["net"] == "latent":
        z, h = net.encode(inp["x"])
        dec = net.decode(refs["encode"].float(), h)
        torch.cuda.synchronize()
        for key, got, ref in (("c4-encode", z, refs["encode"]), ("c4-decode", dec, refs["decode"])):
            wrong += [(key, label, _ratio(key, prec, _stats(got, w))) for label, w in _wrong_refs(c, ref)]
            results.append((key, key, _stats(got, ref)))
    else:
        key = c["key"]
        gots = [net(x, inp["mu"], ts[0] if len(set(ts)) == 1 else ts) for _, ts, x in inp["calls"]]
        torch.cuda.synchronize()
        k = c["ts"].index(c["tpm"])
        wrong = [(key, label, _ratio(key, prec, _stats(gots[k], w))) for label, w in _wrong_refs(c, refs["calls"][k], refs)]
        results = [(key, label, _stats(got, ref)) for (label, _, _), got, ref in zip(inp["calls"], gots, refs["calls"])]
        steps = _step_check(lib, c, net, inp, refs, dev)
    torch.cuda.synchronize()
    lib_bytes = int(net._ctx.L.irsde_device_bytes(net._ctx.h))
    peak = max(refs["peak"], torch.cuda.max_memory_reserved() + lib_bytes)
    seconds = time.perf_counter() - t0
    net._ctx.close()
    del net
    with capsys.disabled():
        print("\n  %s %s: peak %s (library %s), oracle %.1f s, network %.1f s" % (
            c["name"], prec, _gb(peak), _gb(lib_bytes), refs["seconds"], seconds))
        for key, label, s in results:
            print("    %-10s %-34s max %.3e  rms %.3e  cell ratio %6.2f  -> %.3f of the bound" % (
                key, label, s["max"], s["rms"], s["cell"], _ratio(key, prec, s)))
        for key, label, r in wrong:
            print("    %-10s wrong reference: %-30s %.3g x the bound" % (key, label, r))
        for t, r, w in steps:
            print("    step t=%-4d %.3f of the bound; wrong: %s" % (t, r, ", ".join("%s %.3g" % kv for kv in w)))
    for key, label, r in wrong:
        assert r > 1.0, ("the bound does not see a wrong reference", key, label, r)
    for t, r, w in steps:
        for label, rw in w:
            assert rw > 1.0, ("the step bound does not see a wrong reference", t, label, rw)
    assert peak <= c["need"], (peak, c["need"])
    for key, label, s in results:
        assert _ratio(key, prec, s) <= 1.0, (key, label, s)
    for t, r, _ in steps:
        assert r <= 1.0, ("step", t, r)


# ------------------------------------------------------------------------------------------------------------------
# programmatic dependent launch
# ------------------------------------------------------------------------------------------------------------------
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PDL_NEED = 12 * GB


def _pdl_child(out_path):
    """Run in a fresh process: the c2 bf16 forward, a 3-step graph chain of it and the c4 NAFNet bf16 forward."""
    import irsde_b200
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(11)
    net = irsde_b200.ConditionalUNet(3, 3, 64, depth=4, precision="bf16")
    net.load_state_dict(O.make_weights(3, 3, 64, 4, seed=0), strict=True)
    net = net.to(dev)
    mu = torch.rand(8, 3, 256, 256, generator=g).to(dev)
    x = (mu.cpu() + torch.randn(8, 3, 256, 256, generator=g) * (10 / 255)).to(dev)
    zs = torch.randn(3, 8, 3, 256, 256, generator=g).to(dev)
    out = {"c2 forward": net(x, mu, [100, 50, 1, 73, 2, 99, 51, 10])}
    sde = irsde_b200.IRSDE(10, 100, schedule="cosine", eps=0.005, device=dev)
    sde.set_model(net)
    sde.set_mu(mu)
    sde.use_graph = True
    out["c2 3-step graph chain"] = sde.reverse_sde(x, T=3, zs=zs)
    naf = irsde_b200.ConditionalNAFNet(latent=True, precision="bf16", **NAF)
    naf.load_state_dict(O.make_nafnet_weights(4, 64, 1, NAF["enc_blk_nums"], NAF["dec_blk_nums"], seed=6), strict=True)
    naf = naf.to(dev)
    lq = torch.rand(16, 4, 128, 128, generator=g).to(dev)
    out["c4 nafnet forward"] = naf(lq + 0.1, lq, 100)
    torch.cuda.synchronize()
    torch.save({k: v.cpu() for k, v in out.items()}, out_path)


@pytest.mark.gpu
def test_pdl_results_bit_identical(tmp_path, capsys):
    """IRSDE_PDL=1 against IRSDE_PDL=0, each in its own process."""
    _dev()
    free, _ = torch.cuda.mem_get_info()
    if free < PDL_NEED:
        pytest.skip("needs %d bytes of device memory, %d free" % (PDL_NEED, free))
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    res = {}
    for pdl in ("0", "1"):
        path = str(tmp_path / ("pdl%s.pt" % pdl))
        code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_workload_networks as m; m._pdl_child(%r)"
                % (ROOT, tests_dir, path))
        env = dict(os.environ, IRSDE_PDL=pdl)
        flags = ["-s"] if sys.flags.no_user_site else []
        t0 = time.perf_counter()
        p = subprocess.run([sys.executable] + flags + ["-c", code], env=env, cwd=ROOT, capture_output=True, text=True,
                           timeout=900)
        assert p.returncode == 0, (pdl, p.stdout[-2000:], p.stderr[-4000:])
        res[pdl] = torch.load(path, weights_only=True)
        with capsys.disabled():
            print("\n  IRSDE_PDL=%s: %.1f s" % (pdl, time.perf_counter() - t0), end="")
    for k, a in res["0"].items():
        b = res["1"][k]
        assert torch.isfinite(a).all() and a.abs().max().item() > 0, k
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (k, (a - b).abs().max().item())
