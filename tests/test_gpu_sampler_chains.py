"""Every sampler chain a shipped test config or a benchmark workload runs, at its real length, on its real network,
against the oracle run in float64 on the GPU at every time step.

A chain is T network forwards and T fused updates, replayed from one captured step graph.  It reads state that the
per-forward tests never reach: the time embedding comes from the plan's chain table (one row per t, built for all T + 1
rows of the schedule, reallocated and every captured graph dropped when T + 1 passes its capacity of 128), and t, the
index of z and the Philox keys come from the device StepState that set_step starts and advance_step moves.  That state
does not depend on the image size, so every case runs its real architecture on a small ragged batch, B = 2 at
37x53: it needs a pad, its element count leaves a scalar tail in the update kernel, and the fp64 oracle can afford a
forward at every t.

Each case is one (sampler, max_sigma, T, schedule, eps, mode, start T) of a test yml or a bench.WORKLOADS entry:

  network                          sampler                 chains
  ConditionalUNet nf64 d4          IRSDE cosine eps .005   s10 T100 sde (c2/c3, deblurring), s10 T100 posterior
                                                           (deraining), s30 T100 sde (inpainting, sisr), s10 T400
                                                           posterior (c5), s10 T100 ode
  ConditionalUNet nf32 d5          IRSDE                   s30 T100 sde (deshadow)
  ConditionalNAFNet w64 3ch        IRSDE                   s50 T100 sde (refusion.yml x5, latent-dehazing nasde.yml)
  ConditionalNAFNet w64 4ch latent IRSDE                   s50 T200 sde (c4)
  DenoisingUNet nf64 d4            DenoisingSDE            s75 T100 sde; ode from get_optimal_timestep(15) = 14
  DenoisingNAFNet w64              DenoisingSDE            s70 T1000 ode over all 1000 steps; ode and sde from 158
  ConditionalUNet nf64 d4          IRSDE                   s10 T = 127, 128, 129 sde (the chain table's capacity edge)

Every case runs in fp32 and bf16; c2, c5 and c4 also in fp32x3.  Checks of each case:

1. The chain is the loop.  reverse_* with graph replay and without must equal, bit for bit, a stepwise loop of
   noise_fn(x, t) and the public step: with explicit zs (irsde_step), and with the in-kernel Philox (irsde_step_philox)
   keyed by image_base = 5 and then by explicit 64-bit uids.  The loop records every x_t and every noise estimate.
2. Every step against fp64, teacher-forced on the device's own trajectory.  For every t from the start down to 1:
   noise_fn(x_t, t) against the oracle's float64 forward at x_t (max|err| / max|ref|; bf16 also RMS(err) / RMS(ref)),
   and the device's x_{t-1} against the oracle's float64 step from x_t fed the device's noise estimate and the same z
   (the numpy Philox at stream t for the Philox trajectories).  The step bound is STEP_BOUND x what fp32 torch gets on
   the same step, plus, for Philox, the accuracy of the device's normals (2^-19 (1 + |z|) times d step / d z).
3. Before any output is accepted the bounds reject, at t = start, 127, 128 and 129 where the start is >= 129, one middle
   t and t = 1: the oracle forward at t - 1 and t + 1 (a shifted chain-table row), the step coefficients of t - 1 and
   t + 1, the z of step i - 1 and i + 1 (Philox: stream t - 1 and t + 1), and z rolled by one image.  The posterior's
   std at t = 1 does not depend on z, so its z mutations are skipped there.  In bf16 the shifted forward rows are
   printed, not required (see BF16_EVERY below).
4. Free running: x0 of the fp32 and fp32x3 graph chains against the oracle's float64 reverse_chain with the same zs,
   relative to max|x0|, bounded by FREE.  bf16 is printed only.

Measured on an H100 80GB HBM3 at 700 W (fwd = the largest max|err| / max|ref| of the noise estimate over the chain;
bf16 = the largest forward ratio to the bf16 bounds; step = the largest step ratio over the trajectories and
precisions; free = free-running max|err| / max|x0|; wall = fp32 / fp32x3 / bf16 in seconds, the fp64 oracle included):

  case                          fp32 fwd  fp32x3 fwd  bf16   step  free fp32  free fp32x3  free bf16  wall
  d4 s10 T100 sde               6.6e-6    7.3e-6      0.37   0.30  1.2e-6     6.1e-6       7.3e-3     22 / 10 / 8
  d4 s10 T100 posterior         8.6e-6    -           0.50   0.29  1.4e-6     -            8.0e-3     21 / - / 9
  d4 s30 T100 sde               8.1e-6    -           0.41   0.28  1.0e-6     -            9.2e-3     22 / - / 9
  d4 s10 T400 posterior         9.4e-6    8.1e-6      0.46   0.25  2.4e-6     4.8e-6       7.6e-3     74 / 34 / 26
  d4 s10 T100 ode               7.4e-6    -           0.37   0.25  1.1e-6     -            5.4e-3     15 / - / 7
  d5 s30 T100 sde               5.6e-6    -           0.35   0.37  9.4e-7     -            9.3e-3     23 / - / 9
  naf3 s50 T100 sde             1.1e-5    -           0.66   0.32  3.4e-5     -            1.6e-1     16 / - / 8
  naf4 s50 T200 sde             2.9e-5    2.9e-5      0.70   0.33  2.9e-5     2.7e-5       7.3e-2     26 / 16 / 15
  dunet s75 T100 sde            7.4e-6    -           0.47   0.31  1.1e-6     -            2.2e-2     23 / - / 9
  dunet s75 T100 ode from 14    9.6e-6    -           0.46   0.21  4.1e-7     -            1.8e-3     6 / - / 4
  dnaf s70 T1000 ode            2.7e-4    -           0.55   0.24  2.2e-6     -            5.4e-3     76 / - / 40
  dnaf s70 T1000 ode from 158   1.8e-5    -           0.63   0.22  1.2e-6     -            4.5e-3     16 / - / 9
  dnaf s70 T1000 sde from 158   7.4e-5    -           0.69   0.27  1.9e-6     -            5.8e-3     23 / - / 11
  d4 s10 T127 sde               5.9e-6    -           0.36   0.27  9.2e-7     -            4.5e-3     29 / - / 6
  d4 s10 T128 sde               7.3e-6    -           0.36   0.26  1.6e-6     -            7.8e-3     25 / - / 7
  d4 s10 T129 sde               1.2e-5    -           0.45   0.33  1.3e-6     -            7.5e-3     27 / - / 7
  TiledRefusion corner tiles    3.6e-5    -           0.98   0.27  -          -            -          16 / - / 7

The bf16 column and the corner tiles are against the bounds before the last widening of the latent NAFNet's (its
8x24 corner tiles, padded to 16x32, reach 0.89 of the old fp32 bound and 0.98 of the old bf16 ones).  Peak device memory
is at most 4.2 GB.  The 35 chain cases, the two shared-network tests (41 s and 18 s) and the two TiledRefusion tests
run in about 12 minutes.

The bounds are these values with a margin of 1.4x to 3x (the fp32 forward of the T = 1000 NAFNet, whose error grows
with t through the fp32 time embedding, at 1.46x; the T = 127 / 128 / 129 free-running bounds were set from the T = 100
sde chain's value before they were measured, and are 6x to 11x their measurement).  The bf16 forward is checked at every 4th t and at the mutation t's (about 40 s
of fp64 oracle per precision at T = 1000); every step is checked at every t in every precision.

Free-running amplification: the per-step differences are not amplified here.  Relative to max|x0|, the fp32 x0 error
over the largest per-forward error is 0.18 at T = 100 (c2's chain; 3.1 for the Refusion NAFNet), 1.0 at T = 200
(c4), 0.26 at T = 400 (c5) and 0.008 at T = 1000, so every fp32 and fp32x3 chain is bounded.  In bf16 x0 moves by
2e-3 to 0.16 of max|x0|, which is printed only.

Every wrong reference lands past its bound except one class: in bf16 the oracle at t - 1 or t + 1 moves a random-weight
NAFNet's noise estimate by only 0.09 to 0.11 of the bf16 bound at t = 1, and a UNet's by 0.9 to 2.2 of it, so in bf16
those are printed, not required.  In fp32 and fp32x3 they land 5x (the latent NAFNet, before its bound was widened by
1.5x) to thousands of times past.  The closest step mutation is the Philox stream t + 1 at t = 1 of the T = 200 chain
(1.25x); the rest are 1.8x and more.

Three deliberate breaks of the library were tried, and check 1 fails on each: ensure_chain_table writing time t + 1 into
rows >= 128 (T = 128 and 129: the graph chain differs from the loop by 0.68 and 1.17), one_step launching advance_step
before the update (c2's chain: the last update reads row 0, and x0 fails the finite-and-changed check), and set_step starting the z index
at 1 (c2's chain differs from the loop by 13.5).

The other GPU tests: samplers of different lengths sharing one network across the capacity edge (each result equal, bit
for bit, to the same sampler on a freshly built network), and TiledRefusion at the c4 sampler on a latent whose tile edge
leaves four tile shapes (four plans and four chain tables in one context), equal tile by tile to the stepwise Philox
loop keyed by each tile's uid, with the corner-tile group teacher-forced against fp64 at every t.  The CPU test checks
that every sampler of the staged test ymls and of the benchmark workloads is named by a case or listed as unsupported.
"""
import ctypes
import time

import pytest
import torch

import _nafnet_denoising_oracle as DN
from oracle import irsde_oracle as O
from test_gpu_nafnet_kernels import SEED, _z
from test_gpu_task_networks import NAF, UNSUPPORTED, _test_ymls, _yml_networks
from test_gpu_workload_networks import GB, STEP_BOUND, U, _dev, _gb, _oracle64, _to64, _times64, _x_t
from test_gpu_workload_networks import budget, lib  # noqa: F401  (fixtures)

B, H, W = 2, 37, 53
BASE = 5
UIDS = [(7 << 32) | 3, 0x123456789]     # high halves non-zero, out of order
Z_ACC = 2.0 ** -19                       # accuracy of the device's Philox normals, relative to 1 + |z|

# forward bounds per network and precision: fp32 / fp32x3 max|err| / max|ref|; bf16 (max, rms)
FWD = {
    "d4": {"fp32": 2e-5, "fp32x3": 2e-5, "bf16": (6e-2, 4e-2)},
    "d5": {"fp32": 1.5e-5, "fp32x3": 1.5e-5, "bf16": (6e-2, 4e-2)},
    "naf3": {"fp32": 2.5e-5, "fp32x3": 2.5e-5, "bf16": (8e-2, 6e-2)},
    "naf4": {"fp32": 6e-5, "fp32x3": 6e-5, "bf16": (1.2e-1, 9e-2)},   # covers TiledRefusion's 8x24 corner tiles
    "dunet": {"fp32": 2e-5, "fp32x3": 2e-5, "bf16": (6e-2, 4e-2)},
    # fp32 up to t = 1000: the fp32 time embedding's phase error grows with t (test_gpu_task_networks)
    "dnaf": {"fp32": 4e-4, "fp32x3": 4e-4, "bf16": (1e-1, 8e-2)},
}
BF16_EVERY = 4   # bf16 checks the forward at every 4th t and at the mutation t's (the step at every t)
# In bf16 the oracle one row off moves the noise estimate by about what a bf16 forward resolves (0.09 to 0.11 of the
# bf16 bound for the NAFNets at t = 1, 0.9 to 2.2 for the UNets): in bf16 the shifted-row references are printed, not
# required.  The rows are pinned in bf16 by check 1 (bit-equal to the per-t forward) and by the fp32 / fp32x3 runs of
# the same chain, where they land 3.5x to thousands of times past the bound.
# free-running x0 bounds (fp32 and fp32x3, max|err| / max|x0|) by case key
FREE = {"d4 s10 T100 sde": 1.5e-5, "d4 s10 T100 posterior": 4e-6, "d4 s30 T100 sde": 3e-6,
        "d4 s10 T400 posterior": 1e-5, "d4 s10 T100 ode": 3e-6, "d5 s30 T100 sde": 3e-6, "naf3 s50 T100 sde": 7e-5,
        "naf4 s50 T200 sde": 6e-5, "dunet s75 T100 sde": 3e-6, "dunet s75 T100 ode from 14": 1.2e-6,
        "dnaf s70 T1000 ode": 6e-6, "dnaf s70 T1000 ode from 158": 3.5e-6, "dnaf s70 T1000 sde from 158": 5e-6,
        "d4 s10 T127 sde": 1e-5, "d4 s10 T128 sde": 1e-5, "d4 s10 T129 sde": 1e-5}


# ------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------
def _case(key, net, kind, ms, T, mode, start=None, fp32x3=False, ymls=(), workloads=(), seed=0, need_gb=6):
    """mode: sde | posterior | ode for IRSDE, dsde_sde | dsde_ode for DenoisingSDE."""
    c = dict(key=key, net=net, kind=kind, ms=ms, T=T, mode=mode, start=start or T, ymls=list(ymls),
             workloads=list(workloads), seed=seed, need=int(need_gb * GB),
             precs=["fp32", "fp32x3", "bf16"] if fp32x3 else ["fp32", "bf16"])
    c["id"] = "%s, %s" % (key, _gb(c["need"]))
    return c


IRSDE_S10 = ["deblurring/options/test/ir-sde.yml"]
REFUSION_YMLS = ["%s/options/test/refusion.yml" % t for t in ("deraining", "deblurring", "deshadow", "inpainting", "sisr")]
CASES = [
    _case("d4 s10 T100 sde", "d4", "irsde", 10, 100, "sde", fp32x3=True, ymls=IRSDE_S10, workloads=["c2", "c3"]),
    _case("d4 s10 T100 posterior", "d4", "irsde", 10, 100, "posterior", ymls=["deraining/options/test/ir-sde.yml"], seed=1),
    _case("d4 s30 T100 sde", "d4", "irsde", 30, 100, "sde", seed=2,
          ymls=["inpainting/options/test/ir-sde.yml", "sisr/options/test/ir-sde.yml"]),
    _case("d4 s10 T400 posterior", "d4", "irsde", 10, 400, "posterior", fp32x3=True, workloads=["c5"], seed=3),
    _case("d4 s10 T100 ode", "d4", "irsde", 10, 100, "ode", seed=4),
    _case("d5 s30 T100 sde", "d5", "irsde", 30, 100, "sde", ymls=["deshadow/options/test/ir-sde.yml"], seed=5),
    _case("naf3 s50 T100 sde", "naf3", "irsde", 50, 100, "sde", seed=6,
          ymls=REFUSION_YMLS + ["latent-dehazing/options/dehazing/test/nasde.yml"]),
    _case("naf4 s50 T200 sde", "naf4", "irsde", 50, 200, "sde", fp32x3=True, workloads=["c4"], seed=7),
    _case("dunet s75 T100 sde", "dunet", "dsde", 75, 100, "dsde_sde", seed=8),
    _case("dunet s75 T100 ode from 14", "dunet", "dsde", 75, 100, "dsde_ode", start=14, seed=9,
          ymls=["denoising-sde/options/test/ir-sde.yml"]),
    _case("dnaf s70 T1000 ode", "dnaf", "dsde", 70, 1000, "dsde_ode", seed=10),
    _case("dnaf s70 T1000 ode from 158", "dnaf", "dsde", 70, 1000, "dsde_ode", start=158, seed=11,
          ymls=["denoising-sde/options/test/refusion.yml"]),
    _case("dnaf s70 T1000 sde from 158", "dnaf", "dsde", 70, 1000, "dsde_sde", start=158, seed=12),
    _case("d4 s10 T127 sde", "d4", "irsde", 10, 127, "sde", seed=13),
    _case("d4 s10 T128 sde", "d4", "irsde", 10, 128, "sde", seed=14),
    _case("d4 s10 T129 sde", "d4", "irsde", 10, 129, "sde", seed=15),
]
PARAMS = [pytest.param(c, p, id="%s-%s" % (c["id"], p)) for c in CASES for p in c["precs"]]

# the denoising-sde test options run reverse_ode from get_optimal_timestep(degradation sigma) (denoising_model.py:163-168)
MODE_NAMES = {"sde": "sde", "posterior": "posterior", "ode": "ode", "dsde_sde": "sde", "dsde_ode": "ode"}
NATIVE = {"sde": "MODE_SDE", "posterior": "MODE_POSTERIOR", "ode": "MODE_ODE", "dsde_sde": "MODE_DSDE_SDE",
          "dsde_ode": "MODE_DSDE_ODE"}
STEP_FN = {  # the oracle's step as f(schedule, x, mu, noise, z, t)
    "sde": O.irsde_sde_step,
    "posterior": O.irsde_posterior_step,
    "ode": lambda s, x, mu, e, z, t: O.irsde_ode_step(s, x, mu, e, t),
    "dsde_sde": lambda s, x, mu, e, z, t: O.dsde_sde_step(s, x, e, z, t),
    "dsde_ode": lambda s, x, mu, e, z, t: O.dsde_ode_step(s, x, e, t),
}


def _uses_z(mode):
    return mode in ("sde", "posterior", "dsde_sde")


def _schedule(kind, ms, T):
    return O.Schedule(ms, T, "cosine", 0.005) if kind == "irsde" else O.Schedule(ms, T, kind="dsde")


def _sampler_key(kind, ms, T, mode, start):
    return (kind, ms, T, "cosine", 0.005 if kind == "irsde" else 0.04, MODE_NAMES[mode], start)


def _mutation_ts(start):
    ts = {start, max(1, start // 2), 1}
    if start >= 129:
        ts |= {127, 128, 129}
    return ts


# ------------------------------------------------------------------------------------------------------------------
# CPU: every sampler of the test configs and the benchmark is a case or unsupported
# ------------------------------------------------------------------------------------------------------------------
def _yml_sampler(opt, rel):
    """The sampler key a test yml runs, or None when it runs no sampler."""
    sde = opt.get("sde")
    if sde is None:
        return None
    if rel.startswith("denoising-sde/"):
        sc = O.Schedule(sde["max_sigma"], sde["T"], sde.get("schedule", "cosine"), kind="dsde")
        return ("dsde", sde["max_sigma"], sde["T"], sde.get("schedule", "cosine"), 0.04, "ode",
                O.get_optimal_timestep(sc, opt["degradation"]["sigma"]))
    return ("irsde", sde["max_sigma"], sde["T"], sde.get("schedule", "cosine"), sde.get("eps", 0.01),
            sde.get("sampling_mode", "sde"), sde["T"])


def _bench_samplers():
    import bench
    return {name: ("irsde", w["max_sigma"], w["T"], "cosine", w["eps"], w["mode"], w["T"])
            for name, w in bench.WORKLOADS.items() if "plumbing check" not in w["desc"]}


def _uncovered(ymls, cases):
    keyed = lambda c: _sampler_key(c["kind"], c["ms"], c["T"], c["mode"], c["start"])
    missing = []
    for rel, path in sorted(ymls.items()):
        if rel in UNSUPPORTED:
            continue
        opt, _ = _yml_networks(path)
        want = _yml_sampler(opt, rel)
        if want is not None and not any(keyed(c) == want for c in cases if rel in c["ymls"]):
            missing.append((rel, want))
    for name, want in sorted(_bench_samplers().items()):
        if not any(keyed(c) == want for c in cases if name in c["workloads"]):
            missing.append(("bench.WORKLOADS[%r]" % name, want))
    return missing


def test_every_sampler_chain_is_covered():
    ymls = _test_ymls()
    assert len(ymls) >= 15, sorted(ymls)
    named = {y for c in CASES for y in c["ymls"]}
    assert not named - set(ymls), ("cases name configs the reference does not have", sorted(named - set(ymls)))
    assert not named & set(UNSUPPORTED), sorted(named & set(UNSUPPORTED))
    assert {w for c in CASES for w in c["workloads"]} == set(_bench_samplers())
    assert not _uncovered(ymls, CASES), ("samplers neither covered by a case nor unsupported", _uncovered(ymls, CASES))
    # the guard sees a deleted case: every case that stands for a config or a workload is the only one that does
    for c in CASES:
        if c["ymls"] or c["workloads"]:
            assert _uncovered(ymls, [d for d in CASES if d is not c]), ("dropping it goes unnoticed", c["key"])


# ------------------------------------------------------------------------------------------------------------------
# networks, inputs and the oracle
# ------------------------------------------------------------------------------------------------------------------
ENC, DEC = NAF["enc_blk_nums"], NAF["dec_blk_nums"]


def _weights(net, seed):
    if net == "d4":
        return O.make_weights(3, 3, 64, 4, seed=seed)
    if net == "d5":
        return O.make_weights(3, 3, 32, 5, seed=seed)
    if net == "dunet":
        return O.make_weights(3, 3, 64, 4, variant="denoising", seed=seed)
    if net == "naf3":
        return O.make_nafnet_weights(3, 64, 1, ENC, DEC, seed=seed)
    if net == "naf4":
        return O.make_nafnet_weights(4, 64, 1, ENC, DEC, seed=seed)
    return DN.make_weights(3, 64, 1, ENC, DEC, seed=seed)


def _channels(net):
    return 4 if net == "naf4" else 3


def _net(lib, net, prec, P, dev):
    if net == "d4":
        m = lib.ConditionalUNet(3, 3, 64, depth=4, precision=prec)
    elif net == "d5":
        m = lib.ConditionalUNet(3, 3, 32, depth=5, precision=prec)
    elif net == "dunet":
        m = lib.DenoisingUNet(3, 3, 64, depth=4, precision=prec)
    elif net in ("naf3", "naf4"):
        m = lib.ConditionalNAFNet(img_channel=_channels(net), latent=net == "naf4", precision=prec, **NAF)
    else:
        m = lib.DenoisingNAFNet(img_channel=3, precision=prec, **NAF)
    m.load_state_dict(P, strict=True)
    return m.to(dev)


def _oracle_fwd(net, P64, dev):
    """fwd(x, mu, t) of the network in float64 on `dev`, one t for every image."""
    if net in ("d4", "d5", "dunet"):
        nf, depth = (32, 5) if net == "d5" else (64, 4)
        v = "denoising" if net == "dunet" else "conditional"
        return lambda x, mu, t: _oracle64(O.unet_forward, P64, x, mu, _times64([t] * x.shape[0], dev), nf, depth, variant=v,
                                          device=dev)
    if net == "dnaf":
        return lambda x, mu, t: _oracle64(DN.forward, P64, x, _times64([t] * x.shape[0], dev), 64, ENC, 1, DEC, device=dev)
    return lambda x, mu, t: _oracle64(O.nafnet_forward, P64, x, mu, _times64([t] * x.shape[0], dev), 64, ENC, 1, DEC,
                                      latent=net == "naf4", device=dev)


def _inputs(c, dev):
    """mu (None for DenoisingSDE), x at the start of the chain and the zs of every step, fp32 on `dev`."""
    g = torch.Generator().manual_seed(300 + c["seed"])
    shape = (B, _channels(c["net"]), H, W)
    mu, x0 = torch.rand(shape, generator=g, dtype=torch.float64), torch.rand(shape, generator=g, dtype=torch.float64)
    n = torch.randn(shape, generator=g, dtype=torch.float64)
    zs = torch.randn((c["start"],) + shape, generator=g)
    sc = _schedule(c["kind"], c["ms"], c["T"])
    xT = _x_t(sc, mu if c["kind"] == "irsde" else x0, x0, n, [c["start"]] * B).float()
    return dict(mu=mu.float().to(dev) if c["kind"] == "irsde" else None, xT=xT.to(dev), zs=zs.to(dev), sc=sc)


_FREE = {}


def _free_oracle(c, inp, dev):
    """x0 of the oracle's float64 chain from the case's x_T with its zs (shared by the precisions of a case)."""
    if c["key"] not in _FREE:
        _FREE.clear()
        t0 = time.perf_counter()
        fwd = _oracle_fwd(c["net"], _to64(_weights(c["net"], c["seed"]), dev), dev)
        mu = inp["mu"].double() if inp["mu"] is not None else None
        x0 = O.reverse_chain(inp["sc"], lambda x, t: fwd(x, mu, t), inp["xT"].double(), mu,
                             inp["zs"].double() if _uses_z(c["mode"]) else None, c["mode"], T=c["start"])
        torch.cuda.synchronize()
        _FREE[c["key"]] = (x0, time.perf_counter() - t0)
    return _FREE[c["key"]]


# ------------------------------------------------------------------------------------------------------------------
# the device chains and the stepwise loop
# ------------------------------------------------------------------------------------------------------------------
def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _bits(t):
    return t.contiguous().view(torch.int32)


def _sampler(lib, kind, ms, T, net, mu, dev):
    sde = lib.IRSDE(ms, T, schedule="cosine", eps=0.005, device=dev) if kind == "irsde" else lib.DenoisingSDE(ms, T, device=dev)
    sde.set_model(net)
    if mu is not None:
        sde.set_mu(mu)
    sde.seed, sde.seed_auto_increment = SEED, False
    return sde


def _set_z_source(sde, zsrc):
    """zsrc: "zs" (explicit, torch order), "none" (ODE), "philox base" or "philox uids"."""
    sde.rng = "philox" if zsrc.startswith("philox") else "torch"
    sde.image_base = BASE if zsrc == "philox base" else 0
    sde.image_uids = list(UIDS) if zsrc == "philox uids" else None


def _chain(sde, mode, xT, start, zs, use_graph):
    sde.use_graph = use_graph
    return getattr(sde, "reverse_" + MODE_NAMES[mode])(xT, T=start, zs=zs)


def _loop(lib, sde, mode, xT, mu, start, zs, zsrc):
    """The stepwise loop: noise_fn(x, t) and the public step.  -> ({t: x_t} for t = start .. 0, {t: noise estimate})."""
    native = getattr(lib._lib, NATIVE[mode])
    ctx = sde._ctx_for(xT)
    B_, C_, H_, W_ = xT.shape
    st = torch.cuda.current_stream().cuda_stream
    sde._apply_image_ids(ctx, B_, st)
    xs, eps = {start: xT}, {}
    x = xT
    for i, t in enumerate(range(start, 0, -1)):
        e = sde.noise_fn(x, t) if mu is not None else sde.model(x, t)
        if zsrc.startswith("philox"):
            nxt = torch.empty_like(x)
            lib._lib.check(ctx.L.irsde_step_philox(ctx.h, native, _ptr(x), _ptr(mu), _ptr(e), t, _ptr(nxt), B_, C_ * H_ * W_,
                                                   SEED, ctypes.c_void_p(st)), ctx.h)
        else:
            nxt = sde._native_step(native, x, mu, e, zs[i] if zsrc == "zs" else None, t)
        eps[t] = e
        x = xs[t - 1] = nxt
    return xs, eps


def _run_all(lib, sde, c, inp):
    """Check 1 on every z source of the case's mode.  -> {zsrc: (xs, eps)} of the loops, and the graph chain's x0."""
    mode, start, mu, xT = c["mode"], c["start"], inp["mu"], inp["xT"]
    out, x0_graph = {}, None
    for zsrc in (["zs", "philox base", "philox uids"] if _uses_z(mode) else ["none"]):
        _set_z_source(sde, zsrc)
        zs = inp["zs"] if zsrc == "zs" else None
        graph = _chain(sde, mode, xT, start, zs, True)
        eager = _chain(sde, mode, xT, start, zs, False)
        xs, eps = _loop(lib, sde, mode, xT, mu, start, zs, zsrc)
        torch.cuda.synchronize()
        assert torch.isfinite(graph).all() and not torch.equal(graph, xT), zsrc
        assert torch.equal(_bits(graph), _bits(xs[0])), ("graph chain != stepwise loop", zsrc,
                                                         (graph - xs[0]).abs().max().item())
        assert torch.equal(_bits(eager), _bits(xs[0])), ("eager chain != stepwise loop", zsrc,
                                                         (eager - xs[0]).abs().max().item())
        out[zsrc] = (xs, eps)
        if zsrc in ("zs", "none"):
            x0_graph = graph
    if "philox base" in out:
        assert not torch.equal(out["philox base"][0][0], out["philox uids"][0][0])
    _set_z_source(sde, "zs")
    return out, x0_graph


# ------------------------------------------------------------------------------------------------------------------
# teacher-forced checks against float64
# ------------------------------------------------------------------------------------------------------------------
def _fwd_ratio(net, prec, got, ref):
    d = got.double() - ref
    mx = d.abs().max().item() / ref.abs().max().item()
    if prec != "bf16":
        return mx / FWD[net][prec]
    rms = (d.pow(2).mean() / ref.pow(2).mean()).sqrt().item()
    return max(mx / FWD[net]["bf16"][0], rms / FWD[net]["bf16"][1])


def _forward_rows(c, prec, fwd, mu, xs, eps):
    """[(t, ratio)] of the noise estimate at every t (every BF16_EVERY-th and the mutation t's in bf16), and
    [(t, wrong label, ratio)] of the shifted-row references."""
    rows, wrong = [], []
    muts = _mutation_ts(c["start"])
    every = BF16_EVERY if prec == "bf16" else 1
    for t in range(c["start"], 0, -1):
        if t % every and t not in muts:
            continue
        ref = fwd(xs[t], mu, t)
        rows.append((t, _fwd_ratio(c["net"], prec, eps[t], ref)))
        if t in muts:
            for t2 in (t - 1, t + 1):
                wrong.append((t, "oracle at t=%d" % t2, _fwd_ratio(c["net"], prec, eps[t], fwd(xs[t], mu, t2))))
    return rows, wrong


def _uids(zsrc, nimg):
    return list(UIDS) if zsrc == "philox uids" else [BASE + b for b in range(nimg)]


def _z_of(zsrc, zs, uids, i, t, shape, dev):
    """The z of step i (at t) that the trajectory used, float64: zs[i], or the numpy Philox at stream t for the images'
    uids.  None for a step index outside the chain."""
    if zsrc == "zs":
        return zs[i].double() if 0 <= i < zs.shape[0] else None
    return _z(SEED, uids, shape[1] * shape[2] * shape[3], t, dev).reshape(shape)


def _step_rows(c, sc, zsrc, zs, uids, mu, xs, eps, dev):
    """[(t, ratio)] of every step and [(t, wrong label, ratio)] of the mutated steps, for one trajectory (uids: those of
    a Philox trajectory)."""
    mode, start = c["mode"], c["start"]
    fn, uses_z = STEP_FN[mode], _uses_z(mode)
    d = lambda a: None if a is None else a.double()
    rows, wrong = [], []
    muts = _mutation_ts(start)
    for i, t in enumerate(range(start, 0, -1)):
        x, got, e = xs[t], xs[t - 1].double(), eps[t]
        shape = tuple(x.shape)
        z = _z_of(zsrc, zs, uids, i, t, shape, dev) if uses_z else None
        step = lambda zz, tt=t: fn(sc, x.double(), d(mu), e.double(), zz, tt)
        ref = step(z)
        err32 = (fn(sc, x, mu, e, None if z is None else z.float(), t).double() - ref).abs().max().item()
        bound = STEP_BOUND * max(err32, U * ref.abs().max().item()) + torch.zeros_like(ref)
        if uses_z and zsrc != "zs":
            bound = bound + (step(torch.ones_like(z)) - step(torch.zeros_like(z))).abs() * Z_ACC * (1 + z.abs())
        r = lambda a: ((got - a).abs() / bound).max().item()
        rows.append((t, r(ref)))
        if t not in muts:
            continue
        for t2 in (t - 1, t + 1):
            if 1 <= t2 <= c["T"]:
                wrong.append((t, "coefficients of t=%d" % t2, r(fn(sc, x.double(), d(mu), e.double(), z, t2))))
        if not uses_z or (mode == "posterior" and t == 1):   # the posterior's std at t = 1 is sqrt(1e-20 dt) max_sigma
            continue
        for k in (-1, 1):
            zk = _z_of(zsrc, zs, uids, i + k, t + k, shape, dev)
            if zk is not None:
                wrong.append((t, ("z of step i%+d" if zsrc == "zs" else "Philox stream t%+d") % k, r(step(zk))))
        wrong.append((t, "z rolled by one image", r(step(torch.roll(z, 1, 0)))))
    return rows, wrong


def _worst(rows):
    return max(rows, key=lambda tr: tr[-1])


def _peak_and_close(nets):
    torch.cuda.synchronize()
    lib_bytes = sum(int(n._ctx.L.irsde_device_bytes(n._ctx.h)) for n in nets)
    peak = torch.cuda.max_memory_reserved() + lib_bytes
    for n in nets:
        n._ctx.close()
    return peak


@pytest.mark.gpu
@pytest.mark.parametrize("case,prec", PARAMS)
def test_sampler_chain_vs_fp64_oracle(lib, case, prec, budget, capsys):
    c = case
    dev = _dev()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    inp = _inputs(c, dev)
    P = _weights(c["net"], c["seed"])
    net = _net(lib, c["net"], prec, P, dev)
    sde = _sampler(lib, c["kind"], c["ms"], c["T"], net, inp["mu"], dev)
    trajs, x0 = _run_all(lib, sde, c, inp)
    t_dev = time.perf_counter() - t0
    # check 2 and 3
    fwd = _oracle_fwd(c["net"], _to64(P, dev), dev)
    primary = "zs" if "zs" in trajs else "none"
    xs, eps = trajs[primary]
    frows, fwrong = _forward_rows(c, prec, fwd, inp["mu"], xs, eps)
    srows, swrong = {}, []
    for zsrc, (xs_, eps_) in trajs.items():
        srows[zsrc], w = _step_rows(c, inp["sc"], zsrc, inp["zs"], _uids(zsrc, B), inp["mu"], xs_, eps_, dev)
        swrong += [(t, "%s: %s" % (zsrc, label), r) for t, label, r in w]
    t_tf = time.perf_counter() - t0 - t_dev
    # check 4
    ref0, t_free = _free_oracle(c, inp, dev)
    free = (x0.double() - ref0).abs().max().item() / ref0.abs().max().item()
    worst_fwd_rel = max(r for _, r in frows) * FWD[c["net"]][prec] if prec != "bf16" else None
    peak = _peak_and_close([net])
    del net, sde
    with capsys.disabled():
        print("\n  %s %s: %.1f s (device chains and loops %.1f s, teacher-forced fp64 %.1f s, free-running fp64 %.1f s), "
              "peak %s" % (c["key"], prec, time.perf_counter() - t0, t_dev, t_tf, t_free, _gb(peak)))
        t, r = _worst(frows)
        print("    forward: worst %.3f of the bound at t=%d" % (r, t))
        for zsrc, rows in srows.items():
            t, r = _worst(rows)
            print("    step (%s): worst %.3f of the bound at t=%d" % (zsrc, r, t))
        for name, w in (("forward", fwrong), ("step", swrong)):
            t, label, r = min(w, key=lambda x: x[2])
            print("    closest wrong %s reference: %s at t=%d, %.3g x the bound" % (name, label, t, r))
        print("    free-running x0: max|err| / max|x0| = %.3e%s%s" % (
            free, "" if prec == "bf16" else " (%.2g x the largest per-forward max error)" % (free / worst_fwd_rel),
            ", %.3f of the bound" % (free / FREE[c["key"]]) if prec != "bf16" and c["key"] in FREE else ", printed only"))
    for t, label, r in (swrong if prec == "bf16" else fwrong + swrong):
        assert r > 1.0, ("the bound does not see a wrong reference", t, label, r)
    assert peak <= c["need"], (peak, c["need"])
    for t, r in frows:
        assert r <= 1.0, ("forward", t, r)
    for zsrc, rows in srows.items():
        for t, r in rows:
            assert r <= 1.0, ("step", zsrc, t, r)
    if prec != "bf16" and c["key"] in FREE:
        assert free <= FREE[c["key"]], ("free-running", free)


# ------------------------------------------------------------------------------------------------------------------
# samplers sharing one network across the chain table's capacity edge
# ------------------------------------------------------------------------------------------------------------------
SHARE_NEED = 6 * GB


def _need(n):
    _dev()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < n:
        pytest.skip("needs %d bytes of device memory, %d free" % (n, free))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_samplers_share_one_network_across_capacity_edge(lib, prec, capsys):
    """One ConditionalUNet: IRSDE T=100 sde, T=400 posterior (the table grows past 128 rows, the graphs are recaptured),
    the first sampler again, then T=129 sde.  One DenoisingNAFNet: DenoisingSDE T=1000 ode over all steps, sde from 158,
    a T=100 sampler (101 rows of the 1001-row table), then ode from 158.  Each result equals, bit for bit, the same
    sampler on a freshly built network with the same weights."""
    _need(SHARE_NEED)
    dev = _dev()
    t0 = time.perf_counter()
    g = torch.Generator().manual_seed(77)
    for net_key, runs in (("d4", [("a", "irsde", 10, 100, "sde", 100), ("b", "irsde", 10, 400, "posterior", 400),
                                  ("a", "irsde", 10, 100, "sde", 100), ("c", "irsde", 10, 129, "sde", 129)]),
                          ("dnaf", [("a", "dsde", 70, 1000, "dsde_ode", 1000), ("a", "dsde", 70, 1000, "dsde_sde", 158),
                                    ("b", "dsde", 75, 100, "dsde_sde", 100), ("a", "dsde", 70, 1000, "dsde_ode", 158)])):
        P = _weights(net_key, 21)
        shared = _net(lib, net_key, prec, P, dev)
        mu = torch.rand(B, 3, H, W, generator=g).to(dev) if net_key == "d4" else None
        samplers = {}
        for name, kind, ms, T, mode, start in runs:
            if name not in samplers:
                samplers[name] = _sampler(lib, kind, ms, T, shared, mu, dev)
            xT = (torch.rand(B, 3, H, W, generator=g) + 0.2 * torch.randn(B, 3, H, W, generator=g)).to(dev)
            zs = torch.randn(start, B, 3, H, W, generator=g).to(dev) if _uses_z(mode) else None
            got = _chain(samplers[name], mode, xT, start, zs, True)
            fresh = _net(lib, net_key, prec, P, dev)
            want = _chain(_sampler(lib, kind, ms, T, fresh, mu, dev), mode, xT, start, zs, True)
            torch.cuda.synchronize()
            fresh._ctx.close()
            assert torch.isfinite(want).all() and not torch.equal(want, xT)
            assert torch.equal(_bits(got), _bits(want)), (net_key, name, kind, ms, T, mode, start,
                                                          (got - want).abs().max().item())
        shared._ctx.close()
    with capsys.disabled():
        print("\n  shared samplers %s: %.1f s" % (prec, time.perf_counter() - t0), end="")


# ------------------------------------------------------------------------------------------------------------------
# TiledRefusion at the c4 sampler
# ------------------------------------------------------------------------------------------------------------------
TILE_NEED = 6 * GB
LAT_H, LAT_W, TILE = 40, 56, 32   # tiles 32x32, 32x24, 8x32 and 8x24


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_tiled_refusion_c4_sampler(lib, prec, capsys):
    """restore_latent at T = 200 on a 2x4x40x56 latent with 32-pixel tiles: four tile shapes, so one context holds four
    plans and four chain tables.  Every tile equals, bit for bit, the stepwise Philox loop keyed by its uid, and the
    corner-tile group is teacher-forced against float64 at every t."""
    _need(TILE_NEED)
    dev = _dev()
    t0 = time.perf_counter()
    P = _weights("naf4", 7)
    net = _net(lib, "naf4", prec, P, dev)
    c = dict(net="naf4", kind="irsde", ms=50, T=200, mode="sde", start=200)
    sde = _sampler(lib, "irsde", 50, 200, net, None, dev)
    z_all = torch.rand(2, 4, LAT_H, LAT_W, generator=torch.Generator().manual_seed(8)).to(dev)
    pipe = lib.TiledRefusion(None, sde, tile=TILE, mode="sde", seed=SEED)
    out = pipe.restore_latent(z_all)
    units, groups = lib.plan_units(2, LAT_H, LAT_W, TILE)
    assert len(groups) == 4, sorted(groups)
    corner = None
    for shape, uids in sorted(groups.items()):
        mu = torch.stack([z_all[units[u][1], :, units[u][2][0]:units[u][2][1], units[u][2][2]:units[u][2][3]]
                          for u in uids]).contiguous()
        sde.rng, sde.image_uids = "philox", list(uids)
        sde.set_mu(mu)
        xT = sde.noise_state(mu)
        xs, eps = _loop(lib, sde, "sde", xT, mu, 200, None, "philox uids")
        torch.cuda.synchronize()
        for row, u in enumerate(uids):
            _, b, (y0, y1, x0, x1) = units[u]
            assert torch.equal(_bits(out[b, :, y0:y1, x0:x1]), _bits(xs[0][row])), (shape, u)
        if corner is None or shape[0] * shape[1] < corner[0][0] * corner[0][1]:
            corner = (shape, uids, mu, xs, eps)
    shape, uids, mu, xs, eps = corner
    fwd = _oracle_fwd("naf4", _to64(P, dev), dev)
    frows, fwrong = _forward_rows(c, prec, fwd, mu, xs, eps)
    srows, swrong = _step_rows(c, _schedule("irsde", 50, 200), "philox uids", None, list(uids), mu, xs, eps, dev)
    peak = _peak_and_close([net])
    with capsys.disabled():
        print("\n  TiledRefusion c4 sampler %s: %.1f s, peak %s, corner tiles %s (uids %s)" % (
            prec, time.perf_counter() - t0, _gb(peak), shape, uids))
        (tf, rf), (ts, rs) = _worst(frows), _worst(srows)
        print("    forward: worst %.3f of the bound at t=%d; step: worst %.3f at t=%d" % (rf, tf, rs, ts))
        t, label, r = min(fwrong + swrong, key=lambda x: x[2])
        print("    closest wrong reference: %s at t=%d, %.3g x the bound" % (label, t, r))
    for t, label, r in (swrong if prec == "bf16" else fwrong + swrong):
        assert r > 1.0, ("the bound does not see a wrong reference", t, label, r)
    assert peak <= TILE_NEED
    for t, r in frows + srows:
        assert r <= 1.0, (t, r)
