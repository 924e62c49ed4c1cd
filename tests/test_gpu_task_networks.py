"""The network of every shipped task config, at its real architecture, against the oracle run in float64 on the GPU, in
all three precisions, at ragged test-set image sizes as well as at sizes that need no pad:

  yml (codes/config/...)                           network                                            inputs
  {deraining,deblurring,inpainting,sisr}/          ConditionalUNet(3, 3, 64, depth=4)                 2x3x321x481, 1x3x720x1280
      options/test/ir-sde.yml
  deshadow/options/test/ir-sde.yml                 ConditionalUNet(3, 3, 32, depth=5)                 2x3x321x481, 1x3x480x640
  denoising-sde/options/test/ir-sde.yml            DenoisingUNet(3, 3, 64, depth=4)                   2x3x321x481, 1x3x512x768
  {deraining,deblurring,deshadow,inpainting,sisr}/ ConditionalNAFNet(3, 64, 1, [1,1,1,28], [1,1,1,1]) 2x3x321x481, 1x3x720x1280
      options/test/refusion.yml
  denoising-sde/options/test/refusion.yml          DenoisingNAFNet(3, 64, 1, [1,1,1,28], [1,1,1,1])   2x3x321x481, 1x3x512x768
  latent-dehazing/options/dehazing/test/nasde.yml  UNet(3, 3, 8, [4,8,8,16], 8) encode / decode and   1x3x750x1000
  (and unet-latent/options/test/test_latent.yml)   the latent ConditionalNAFNet(8, 64, 1, [1,1,1,28]) (latent 1x8x94x126)
                                                   on the whole latent, as that task's test.py runs it

321x481 (Rain100H, CBSD68) is padded by 15 rows and 15 columns to 336x496 (the UNets reflect, the NAFNets zero-pad)
and by 31 / 31 to 352x512 for the depth-5 UNet; its deep levels (42x62, 21x31, 11x16) end conv tiles mid-tile and give
LinearAttention a partial last chunk.  For the latent task, 750x1000 is reflect-padded to 752x1008 by the autoencoder and
its 94x126 latent zero-padded to 96x128 by the NAFNet.  720x1280, 480x640 and 512x768 need no pad.

Each score network runs at t = T, T/2 (158 for T = 1000) and 1, plus one call with a different t per image where B > 1.
Its input is the x_t of the task's schedule, and every sampler step its yml can select (reverse_sde, and
reverse_posterior for deraining; DenoisingSDE's sde and ode) is checked teacher-forced as in test_gpu_workload_networks:
`_native_step` fed the oracle's noise estimate, against the oracle's step in float64.  The autoencoder's decode takes
the oracle's latent and the skips the GPU's own encode left behind.

Statistics (err = network - oracle): max = max|err| / max|ref| and rms = RMS(err) / RMS(ref) over the whole output;
cell = the largest over the median of the (image, 32x32 block) cells' RMS(err), cells covering the whole cropped output
with partial cells at the right and bottom edges, each cell's mean square over its own pixel count; band = RMS(err) over
the last `pad` rows and columns of the output (the pixels next to the padded region) over RMS(err) in the rest.  A size
that is a multiple of the pad step has no band, and its band statistic and the pad-mode and crop-corner wrong references
below are skipped.  fp32 and fp32x3 are bounded by max, bf16 by max, rms, cell and band.

Before any output is accepted, each case shows that its bounds reject wrong references at t = T/2: the batch rolled by
one image, the oracle at t - 1 and t + 1, one 32x32 block read one pixel up in the middle of the last image and in its
bottom-right edge cell, the oracle fed the input pre-padded to the multiple with the other pad mode (zeros for the UNets,
reflect for the NAFNets; the oracle pads nothing more) and cropped, and the bottom-right HxW of the oracle's whole padded
output instead of the top-left.

Measured on an H100 80GB HBM3 at 700 W (the largest over the calls of a case; peak = the largest over the three
precisions; wall = fp64 oracle + the three precisions):

  case                        fp32 max  fp32x3 max  bf16 max  bf16 rms  cell  band  peak     wall
  ir-sde d4 2x321x481         7.8e-6    7.1e-6      2.5e-2    1.23e-2   1.48  0.99  6.1 GB   4.5 + 10.6 s
  ir-sde d4 1x720x1280        1.0e-5    7.1e-6      2.7e-2    2.36e-2   1.17  -     13.6 GB  5.8 + 10.7 s
  deshadow d5 2x321x481       1.2e-5    1.2e-5      3.9e-2    2.09e-2   1.38  1.02  5.0 GB   2.9 + 8.5 s
  deshadow d5 1x480x640       7.1e-6    7.1e-6      2.3e-2    1.18e-2   1.28  -     4.6 GB   2.2 + 8.2 s
  dsde unet 2x321x481         9.4e-6    6.3e-6      2.3e-2    1.98e-2   1.27  1.00  6.1 GB   3.5 + 9.4 s
  dsde unet 1x512x768         8.2e-6    4.9e-6      2.1e-2    1.95e-2   1.13  -     6.7 GB   3.3 + 9.5 s
  refusion 2x321x481          1.7e-5    1.7e-5      3.1e-2    3.43e-2   1.64  1.03  3.2 GB   1.5 + 5.9 s
  refusion 1x720x1280         7.1e-6    6.3e-6      4.1e-2    3.37e-2   1.11  -     6.5 GB   1.9 + 5.8 s
  dsde refusion 2x321x481     1.4e-4    1.4e-4      5.0e-2    5.10e-2   1.94  1.07  3.7 GB   1.3 + 6.0 s
  dsde refusion 1x512x768     5.1e-5    5.1e-5      3.7e-2    3.24e-2   1.09  -     3.9 GB   1.0 + 5.2 s
  latent-dehazing encode      9.7e-7    1.0e-6      6.1e-3    5.43e-3   1.02  -     3.3 GB   1.1 + 4.9 s
  latent-dehazing decode      1.0e-6    2.0e-6      9.2e-3    5.46e-3   1.13  0.95
  latent-dehazing nafnet      5.2e-6    5.3e-6      4.0e-2    3.55e-2   1.07  1.00

The fp32 error of the Denoising NAFNet grows with t: 6.4e-5 at t = 1000 and 1.4e-4 on the t = 700 image of the
per-image call, against 2.0e-5 at t = 1.  It is the accuracy of the fp32 time embedding (sin / cos of t times a
frequency), which the reference computes in fp32 too: the plain fp32 oracle on the CPU is 5.2e-5 off the float64 one on
this network at t = 1000.  In the per-image calls of the score networks the cell ratio compares an image at large t with
one at small t, which is why fp32 cell ratios reach 12 there; only bf16 is bounded by it.  The teacher-forced steps come
to 0.25 of their bound.  The whole file runs in about 130 s.

Every wrong reference lands past its bounds, thousands of times in fp32.  In bf16 the closest are the oracle at t - 1
for the UNets (2.4x to 5.6x the bound) and at least 10x for the NAFNets and the autoencoder.  The input padded the
other way lands 10x to 33x past, with a band statistic of 5.8 to 10.5 for the UNets, 24 for the decode, and 2.0 to 2.5
for the NAFNets: their channel attention pools over the padded region, so a wrong pad moves the whole output.
Three deliberate breaks of the library were tried, and the test fails on each: the tensor-core conv's cropped NCHW head
keeping the bottom-right HxW (ir-sde d4 at 321x481 in bf16: 21x the bound), the NAFNet input packing reflecting instead
of zero-padding (refusion at 321x481: 13x), and the ROWS conv dropping its last partial column of tiles on the
248-pixel-wide level (ir-sde d4 and dsde unet at 321x481: 18x and 27x, cell ratio 40 to 53).

Every case states a device-memory budget (at most 24 GB) in its id and skips when that much is not free; it prints its
peak (torch's reserved peak plus the library's device bytes), its errors and its runtime.

The CPU tests check that every network a task's test options build is a case here or is listed in UNSUPPORTED (they
skip where oracle/_ref is not staged), and that the float64 oracle wrapper agrees with the fp32 CPU oracle on small
configs of the depth-5 UNet, the denoising UNet and NAFNet, the 8-channel latent NAFNet and this autoencoder.
"""
import glob
import math
import os
import time

import pytest
import torch
import torch.nn.functional as F

import _nafnet_denoising_oracle as DN
from oracle import irsde_oracle as O
from test_gpu_workload_networks import (BUDGET, CELL, GB, STEP_BOUND, U, _DtypeAudit, _dev, _gb, _oracle64, _to64,
                                        _times64, _x_t)
from test_gpu_workload_networks import budget, lib  # noqa: F401  (fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_CONFIG = os.path.join(ROOT, "oracle", "_ref", "codes", "config")
PRECISIONS = ["fp32", "fp32x3", "bf16"]

# bounds: the measured values of the module docstring with a margin of 1.4x to 3x
BOUNDS = {   # max32: fp32 / fp32x3 max; bf16: max, rms, cell and band
    "ir-sde d4": dict(max32=2e-5, max=4e-2, rms=3.5e-2, cell=2.2, band=1.5),
    "deshadow d5": dict(max32=2.5e-5, max=5.8e-2, rms=3e-2, cell=2.0, band=1.5),
    "dsde unet": dict(max32=2e-5, max=3.5e-2, rms=3e-2, cell=2.0, band=1.5),
    "refusion": dict(max32=3e-5, max=6e-2, rms=5e-2, cell=2.4, band=1.5),
    # fp32 at t up to 1000: the fp32 time embedding's phase error grows with t (the plain fp32 oracle on the CPU is
    # 5.2e-5 off the float64 one at t = 1000 on this network, 2.2e-6 at t = 1), so the bound covers the t = 700 image
    "dsde refusion": dict(max32=2.5e-4, max=7.5e-2, rms=7.5e-2, cell=2.8, band=1.5),
    "latent-dehazing encode": dict(max32=2e-6, max=9e-3, rms=8e-3, cell=2.0, band=1.5),
    "latent-dehazing decode": dict(max32=4e-6, max=1.4e-2, rms=8e-3, cell=2.0, band=1.5),
    "latent-dehazing nafnet": dict(max32=1e-5, max=6e-2, rms=5e-2, cell=2.0, band=1.5),
}

# test options whose networks this library does not build, by path under codes/config
UNSUPPORTED = {
    "latent-bokeh/options/bokeh/test/refusion.yml":
        "its ConditionalNAFNet adds a lens embedding (cam_mlp) to the time embedding, which is not implemented",
    "stereo-sr/options/ssr/test/refusion.yml":
        "its NAFNet runs SCAM stereo cross-attention between the views after every block, which is not implemented",
}

# reference constructor defaults the ymls may leave out
DEFAULTS = {"ConditionalNAFNet": dict(img_channel=3)}

UNET64 = ("ConditionalUNet", dict(in_nc=3, out_nc=3, nf=64, depth=4))
UNET32D5 = ("ConditionalUNet", dict(in_nc=3, out_nc=3, nf=32, depth=5))
NAF = dict(width=64, middle_blk_num=1, enc_blk_nums=[1, 1, 1, 28], dec_blk_nums=[1, 1, 1, 1])
NAF3 = ("ConditionalNAFNet", dict(img_channel=3, **NAF))
NAF8 = ("ConditionalNAFNet", dict(img_channel=8, **NAF))
AE = ("UNet", dict(in_ch=3, out_ch=3, ch=8, ch_mult=[4, 8, 8, 16], embed_dim=8))
IRSDE_YMLS = ["%s/options/test/ir-sde.yml" % t for t in ("deraining", "deblurring", "inpainting", "sisr")]
REFUSION_YMLS = ["%s/options/test/refusion.yml" % t for t in ("deraining", "deblurring", "deshadow", "inpainting", "sisr")]
LATENT_YMLS = ["latent-dehazing/options/dehazing/test/nasde.yml", "unet-latent/options/test/test_latent.yml"]


def _case(key, need_gb, arch, nets, ymls, B, H, W, sdes, ts=(100, 50, 1), mixed=None, seed=0):
    """sdes: [(kind, max_sigma, T, modes)], the first one gives the x_t of the calls."""
    c = dict(key=key, need=int(need_gb * GB), arch=arch, nets=nets, ymls=ymls, B=B, H=H, W=W, sdes=sdes, ts=list(ts),
             tpm=ts[1], mixed=mixed if B > 1 else None, seed=seed)
    assert c["need"] <= BUDGET
    c["id"] = "%s %dx%dx%d, %s" % (key, B, H, W, _gb(c["need"]))
    return c


IRSDE_D4_SDES = [("irsde", 10, 100, ["sde", "posterior"]), ("irsde", 30, 100, ["sde"])]
CASES = [
    _case("ir-sde d4", 10, "unet", [UNET64], IRSDE_YMLS, 2, 321, 481, IRSDE_D4_SDES, mixed=[73, 2]),
    _case("ir-sde d4", 18, "unet", [UNET64], IRSDE_YMLS, 1, 720, 1280, IRSDE_D4_SDES, seed=1),
    _case("deshadow d5", 8, "unet", [UNET32D5], ["deshadow/options/test/ir-sde.yml"], 2, 321, 481,
          [("irsde", 30, 100, ["sde"])], mixed=[73, 2], seed=2),
    _case("deshadow d5", 8, "unet", [UNET32D5], ["deshadow/options/test/ir-sde.yml"], 1, 480, 640,
          [("irsde", 30, 100, ["sde"])], seed=3),
    _case("dsde unet", 10, "dunet", [UNET64], ["denoising-sde/options/test/ir-sde.yml"], 2, 321, 481,
          [("dsde", 75, 100, ["dsde_sde", "dsde_ode"])], mixed=[73, 2], seed=4),
    _case("dsde unet", 10, "dunet", [UNET64], ["denoising-sde/options/test/ir-sde.yml"], 1, 512, 768,
          [("dsde", 75, 100, ["dsde_sde", "dsde_ode"])], seed=5),
    _case("refusion", 6, "nafnet", [NAF3], REFUSION_YMLS, 2, 321, 481, [("irsde", 50, 100, ["sde"])], mixed=[73, 2],
          seed=6),
    _case("refusion", 10, "nafnet", [NAF3], REFUSION_YMLS, 1, 720, 1280, [("irsde", 50, 100, ["sde"])], seed=7),
    _case("dsde refusion", 6, "dnafnet", [NAF3], ["denoising-sde/options/test/refusion.yml"], 2, 321, 481,
          [("dsde", 70, 1000, ["dsde_sde", "dsde_ode"])], ts=(1000, 158, 1), mixed=[700, 3], seed=8),
    _case("dsde refusion", 6, "dnafnet", [NAF3], ["denoising-sde/options/test/refusion.yml"], 1, 512, 768,
          [("dsde", 70, 1000, ["dsde_sde", "dsde_ode"])], ts=(1000, 158, 1), seed=9),
    _case("latent-dehazing", 6, "latent", [AE, NAF8], LATENT_YMLS, 1, 750, 1000, [("irsde", 50, 100, ["sde"])],
          seed=10),
]


# ------------------------------------------------------------------------------------------------------------------
# CPU: every test config is a case or unsupported; the float64 wrapper on small configs of these networks
# ------------------------------------------------------------------------------------------------------------------
def _test_ymls():
    if not os.path.isdir(REF_CONFIG):
        pytest.skip("the reference is not staged under oracle/_ref")
    paths = sorted(glob.glob(os.path.join(REF_CONFIG, "*", "options", "**", "test", "**", "*.yml"), recursive=True))
    return {os.path.relpath(p, REF_CONFIG): p for p in paths}


def _yml_networks(path):
    """[(key, model, setting with the reference's defaults filled in)] for network_G / network_L of a yml."""
    yaml = pytest.importorskip("yaml")
    with open(path) as f:
        opt = yaml.safe_load(f)
    out = []
    for key in ("network_G", "network_L"):
        if key in opt:
            net = opt[key]
            model = net.get("which_model_G", net.get("which_model"))
            out.append((key, model, dict(DEFAULTS.get(model, {}), **net["setting"])))
    return opt, out


def test_every_task_test_config_is_covered():
    ymls = _test_ymls()
    assert len(ymls) >= 15, sorted(ymls)
    named = {y for c in CASES for y in c["ymls"]}
    assert not named - set(ymls), ("cases name configs the reference does not have", sorted(named - set(ymls)))
    assert not set(UNSUPPORTED) - set(ymls), ("stale UNSUPPORTED entries", sorted(set(UNSUPPORTED) - set(ymls)))
    assert not named & set(UNSUPPORTED), sorted(named & set(UNSUPPORTED))
    missing = []
    for rel, path in ymls.items():
        if rel in UNSUPPORTED:
            continue
        opt, nets = _yml_networks(path)
        assert nets, rel
        cases = [c for c in CASES if rel in c["ymls"]]
        for key, model, setting in nets:
            if not any((model, setting) in c["nets"] for c in cases):
                missing.append((rel, key, model, setting))
        sde = opt.get("sde")
        if sde is not None and nets[0][0] == "network_G":
            want = (sde["max_sigma"], sde["T"])
            if not any((ms, T) == want for c in cases for _, ms, T, _ in c["sdes"]):
                missing.append((rel, "sde", want))
            mode = sde.get("sampling_mode")
            if mode is not None and not any(mode in modes for c in cases for _, ms, T, modes in c["sdes"]
                                            if (ms, T) == want):
                missing.append((rel, "sampling_mode", mode))
    assert not missing, ("test configs neither covered by a case nor listed in UNSUPPORTED", missing)
    with pytest.raises(AssertionError):   # the guard sees a deleted case
        _covered_without(ymls, CASES[-1])


def _covered_without(ymls, dropped):
    for rel, path in ymls.items():
        if rel in UNSUPPORTED:
            continue
        for key, model, setting in _yml_networks(path)[1]:
            assert any((model, setting) in c["nets"] for c in CASES if c is not dropped and rel in c["ymls"]), rel


def test_fp64_oracle_wrapper_matches_fp32_oracle_on_cpu_task_configs():
    """The wrapped oracle on small configs of this file's networks, on the CPU: within fp32 rounding of the plain fp32
    oracle and not equal to it, with every floating-point tensor any torch call returned in float64."""
    cpu = torch.device("cpu")
    g = torch.Generator().manual_seed(1)
    ts = [9, 70]
    x, cond = torch.rand(2, 3, 18, 22, generator=g), torch.rand(2, 3, 18, 22, generator=g)
    runs = []
    P = O.make_weights(3, 3, 4, 5, seed=11)          # depth 5: pad to 32, mid level at H/16
    runs.append(("unet depth 5", lambda P, x, c, t: O.unet_forward(P, x, c, t, 4, 5), P, (x, cond)))
    P = O.make_weights(3, 3, 8, 2, variant="denoising", seed=12)
    runs.append(("denoising unet", lambda P, x, t: O.unet_forward(P, x, None, t, 8, 2, variant="denoising"), P, (x,)))
    P = O.make_nafnet_weights(3, 16, 1, [1, 1], [1, 1], seed=13)
    runs.append(("nafnet", lambda P, x, c, t: O.nafnet_forward(P, x, c, t, 16, [1, 1], 1, [1, 1]), P, (x, cond)))
    P = DN.make_weights(3, 16, 1, [1, 1], [1, 1], seed=14)
    runs.append(("denoising nafnet", lambda P, x, t: DN.forward(P, x, t, 16, [1, 1], 1, [1, 1]), P, (x,)))
    x8, c8 = torch.rand(2, 8, 10, 14, generator=g), torch.rand(2, 8, 10, 14, generator=g)
    P = O.make_nafnet_weights(8, 16, 1, [1, 1], [1, 1], seed=15)   # img_channel 8: 16-channel intro, 8-channel ending
    runs.append(("latent nafnet img 8", lambda P, x, c, t: O.nafnet_forward(P, x, c, t, 16, [1, 1], 1, [1, 1], latent=True),
                 P, (x8, c8)))
    for name, fn, P, args in runs:
        audit = _DtypeAudit()
        with audit:
            y64 = _oracle64(lambda P64, *a: fn(P64, *a, _times64(ts, cpu)), _to64(P, cpu), *args, device=cpu)
        _close(name, audit.seen, y64, fn(P, *args, torch.tensor(ts)))
    P = O.make_latent_unet_weights(3, 3, 2, [4, 8, 8, 16], 8, seed=16)
    xa = torch.rand(1, 3, 37, 45, generator=g)
    audit = _DtypeAudit()
    with audit:
        z64, h64 = _oracle64(O.latent_unet_encode, _to64(P, cpu), xa, [4, 8, 8, 16], device=cpu)
        d64 = _oracle64(O.latent_unet_decode, _to64(P, cpu), z64, h64, [4, 8, 8, 16], 37, 45, device=cpu)
    z32, h32 = O.latent_unet_encode(P, xa, [4, 8, 8, 16])
    _close("latent encode", audit.seen, z64, z32)
    _close("latent decode", audit.seen, d64, O.latent_unet_decode(P, z32, h32, [4, 8, 8, 16], 37, 45))


def _close(name, seen, y64, y32):
    assert seen == {(torch.float64, "cpu")}, (name, seen)
    assert y64.dtype == torch.float64 and y64.shape == y32.shape, name
    d = (y64 - y32.double()).abs().max().item()
    scale = y32.abs().max().item()
    assert 0 < d <= 1e-5 * scale, (name, d, scale)


# ------------------------------------------------------------------------------------------------------------------
# inputs and the oracle's references
# ------------------------------------------------------------------------------------------------------------------
def _schedule(kind, max_sigma, T):
    return O.Schedule(max_sigma, T, "cosine", 0.005) if kind == "irsde" else O.Schedule(max_sigma, T, kind="dsde")


def _pad_step(c, part):
    """(multiple the network pads to, its pad mode, the other mode) of a case's network."""
    if c["arch"] in ("unet", "dunet"):
        return 2 ** c["nets"][0][1]["depth"], "reflect", "constant"
    if part == "encode":
        return 2 ** len(AE[1]["ch_mult"]), "reflect", "constant"
    return 2 ** len(NAF["enc_blk_nums"]), "constant", "reflect"


def _prepad(x, s, mode):
    if x is None:
        return None
    H, W = x.shape[2:]
    return F.pad(x, (0, (s - W % s) % s, 0, (s - H % s) % s), mode)


def _weights(c):
    s, a = c["seed"], c["arch"]
    if a in ("unet", "dunet"):
        n = c["nets"][0][1]
        return O.make_weights(3, 3, n["nf"], n["depth"], variant="conditional" if a == "unet" else "denoising", seed=s)
    if a == "nafnet":
        return O.make_nafnet_weights(3, 64, 1, NAF["enc_blk_nums"], NAF["dec_blk_nums"], seed=s)
    if a == "dnafnet":
        return DN.make_weights(3, 64, 1, NAF["enc_blk_nums"], NAF["dec_blk_nums"], seed=s)
    return O.make_latent_unet_weights(seed=s, **AE[1]), O.make_nafnet_weights(8, 64, 1, NAF["enc_blk_nums"],
                                                                              NAF["dec_blk_nums"], seed=s + 1)


def _oracle_fn(c, P64, dev):
    """fwd(x, mu, ts) of the case's score network in float64 on `dev`."""
    a = c["arch"]
    if a in ("unet", "dunet"):
        n = c["nets"][0][1]
        v = "conditional" if a == "unet" else "denoising"
        return lambda x, mu, ts: _oracle64(O.unet_forward, P64, x, mu, _times64(ts, dev), n["nf"], n["depth"], variant=v,
                                           device=dev)
    if a == "dnafnet":
        return lambda x, mu, ts: _oracle64(DN.forward, P64, x, _times64(ts, dev), 64, NAF["enc_blk_nums"], 1,
                                           NAF["dec_blk_nums"], device=dev)
    return lambda x, mu, ts: _oracle64(O.nafnet_forward, P64, x, mu, _times64(ts, dev), 64, NAF["enc_blk_nums"], 1,
                                       NAF["dec_blk_nums"], latent=a == "latent", device=dev)


def _score_refs(c, part, fwd, calls, mu, refs):
    """The oracle at every call, at t = T/2 -+ 1, with the wrong pad mode and cropped from the wrong corner."""
    k = c["ts"].index(c["tpm"])
    s, right, wrong = _pad_step(c, part)
    _, _, H, W = calls[k][2].shape
    out = []
    for i, (_, ts, x) in enumerate(calls):
        if i == k and (H % s or W % s):
            # the input pre-padded the oracle's own way is the oracle's own forward: its top-left HxW is the reference
            full = fwd(_prepad(x, s, right), _prepad(mu, s, right), ts)
            out.append(full[..., :H, :W])
            refs["crop corner"] = full[..., -H:, -W:]
            refs["pad mode"] = fwd(_prepad(x, s, wrong), _prepad(mu, s, wrong), ts)[..., :H, :W]
            del full
        else:
            out.append(fwd(x, mu, ts))
    x = calls[k][2]
    B = x.shape[0]
    refs["t-1"] = fwd(x, mu, [c["tpm"] - 1] * B)
    refs["t+1"] = fwd(x, mu, [c["tpm"] + 1] * B)
    return out


def _calls(c, g, shape, mu, dev):
    """[(label, ts, x_t)] at each t of the case (and per-image ts), the x_t of its first sde; mu None for DenoisingSDE
    (x_t = x0 + sigmā_t n there).  Also returns z and the schedule."""
    kind, ms, T, _ = c["sdes"][0]
    sc = _schedule(kind, ms, T)
    if c["arch"] == "latent":   # the clean latent near the hazy one
        x0 = mu + 0.2 * torch.randn(shape, generator=g, dtype=torch.float64)
    else:
        x0 = torch.rand(shape, generator=g, dtype=torch.float64)
    n, z = torch.randn(shape, generator=g, dtype=torch.float64), torch.randn(shape, generator=g, dtype=torch.float64)
    m = x0 if mu is None else mu
    tss = [[t] * shape[0] for t in c["ts"]] + ([list(c["mixed"])] if c["mixed"] else [])
    calls = [("t=%s" % (ts[0] if len(set(ts)) == 1 else ts), ts, _x_t(sc, m, x0, n, ts).float().to(dev)) for ts in tss]
    return calls, z.float().to(dev)


_REFS = {}


def _oracle_refs(c, dev):
    """The oracle's outputs of a case (computed once, shared by the three precisions), with its own peak and time."""
    if c["id"] in _REFS:
        return _REFS[c["id"]]
    _REFS.clear()   # one case's references at a time
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator().manual_seed(200 + c["seed"])
    B, H, W = c["B"], c["H"], c["W"]
    refs = {}
    if c["arch"] == "latent":
        Pa, Pn = _weights(c)
        P64 = _to64(Pa, dev)
        ch_mult = AE[1]["ch_mult"]
        img = torch.rand(B, 3, H, W, generator=g).to(dev)
        z, h = _oracle64(O.latent_unet_encode, P64, img, ch_mult, device=dev)
        s, right, wrong = _pad_step(c, "encode")
        enc = dict(img=img, ref=z, wrongs={})
        enc["wrongs"]["pad mode"], hw = _oracle64(O.latent_unet_encode, P64, _prepad(img, s, wrong), ch_mult, device=dev)
        Hp, Wp = img.shape[2] + (-H) % s, img.shape[3] + (-W) % s
        dec = dict(ref=_oracle64(O.latent_unet_decode, P64, z, h, ch_mult, H, W, device=dev), wrongs={})
        dec["wrongs"]["pad mode"] = _oracle64(O.latent_unet_decode, P64, z, hw, ch_mult, H, W, device=dev)
        dec["wrongs"]["crop corner"] = _oracle64(O.latent_unet_decode, P64, z, h, ch_mult, Hp, Wp, device=dev)[..., -H:, -W:]
        del h, hw, P64
        refs["encode"], refs["decode"] = enc, dec
        mu = z.float().double().cpu()
        calls, zz = _calls(c, g, tuple(mu.shape), mu, dev)
        mu = mu.float().to(dev)
        P64 = _to64(Pn, dev)
    else:
        shape = (B, 3, H, W)
        mu = torch.rand(shape, generator=g, dtype=torch.float64) if c["arch"] in ("unet", "nafnet") else None
        calls, zz = _calls(c, g, shape, mu, dev)
        mu = mu.float().to(dev) if mu is not None else None
        P64 = _to64(_weights(c), dev)
    score = dict(calls=calls, mu=mu, z=zz, wrongs={})
    score["refs"] = _score_refs(c, "score", _oracle_fn(c, P64, dev), calls, mu, score["wrongs"])
    refs["score"] = score
    torch.cuda.synchronize()
    del P64
    refs["peak"] = torch.cuda.max_memory_reserved()
    refs["seconds"] = time.perf_counter() - t0
    torch.cuda.empty_cache()
    _REFS[c["id"]] = refs
    return refs


# ------------------------------------------------------------------------------------------------------------------
# error statistics and bounds
# ------------------------------------------------------------------------------------------------------------------
def _cells(err, ref):
    """RMS(err) in each (image, 32x32 block) cell over all channels, partial cells at the right and bottom edges each
    over its own pixel count, divided by RMS(ref) over the whole output."""
    B, C, H, W = err.shape
    ph, pw = (-H) % CELL, (-W) % CELL
    e2 = F.pad(err.double().pow(2).sum(1), (0, pw, 0, ph))
    e2 = e2.reshape(B, (H + ph) // CELL, CELL, (W + pw) // CELL, CELL).sum(dim=(2, 4))
    n = F.pad(torch.ones(1, H, W, dtype=torch.float64, device=err.device), (0, pw, 0, ph))
    n = n.reshape(1, (H + ph) // CELL, CELL, (W + pw) // CELL, CELL).sum(dim=(2, 4)) * C
    return (e2 / n).sqrt() / ref.double().pow(2).mean().sqrt()


def _band(err, pad):
    """RMS(err) over the last pad[0] rows and pad[1] columns over RMS(err) in the rest; None without a pad."""
    if pad == (0, 0):
        return None
    H, W = err.shape[2:]
    m = torch.zeros(H, W, dtype=torch.bool, device=err.device)
    m[H - pad[0]:, :] = pad[0] > 0
    m[:, W - pad[1]:] |= pad[1] > 0
    e2 = err.double().pow(2).mean(dim=(0, 1))
    return (e2[m].mean() / e2[~m].mean()).sqrt().item()


def _stats(got, ref, pad):
    d = got.double() - ref
    cells = _cells(d, ref)
    med = cells.median().item()
    return dict(max=d.abs().max().item() / ref.abs().max().item(),
                rms=(d.pow(2).mean() / ref.pow(2).mean()).sqrt().item(),
                cell=cells.max().item() / med if med > 0 else math.inf, band=_band(d, pad))


def _ratio(key, prec, s):
    """Largest statistic / its bound: <= 1 passes."""
    b = BOUNDS[key]
    if prec != "bf16":
        return s["max"] / b["max32"]
    r = max(s["max"] / b["max"], s["rms"] / b["rms"], s["cell"] / b["cell"])
    return r if s["band"] is None else max(r, s["band"] / b["band"])


def _shift_cell(ref, b, y0, x0):
    """ref with the (partial) 32x32 cell at (y0, x0) of image b read one pixel up."""
    r = ref.clone()
    h, w = min(CELL, ref.shape[2] - y0), min(CELL, ref.shape[3] - x0)
    r[b, :, y0:y0 + h, x0:x0 + w] = ref[b, :, y0 - 1:y0 - 1 + h, x0:x0 + w]
    return r


def _wrong_refs(ref, wrongs):
    """[(label, wrong reference)] for one output."""
    B, H, W = ref.shape[0], ref.shape[2], ref.shape[3]
    out = [("middle block read a pixel up", _shift_cell(ref, B - 1, max(1, H // CELL // 2) * CELL,
                                                            max(1, W // CELL // 2) * CELL)),
           ("bottom-right edge cell read a pixel up", _shift_cell(ref, B - 1, (H - 1) // CELL * CELL,
                                                                  (W - 1) // CELL * CELL))]
    if B > 1:
        out.append(("batch rolled by one image", torch.roll(ref, 1, dims=0)))
    labels = {"t-1": "oracle at t-1", "t+1": "oracle at t+1", "pad mode": "input padded the other way",
              "crop corner": "cropped from the bottom-right"}
    return out + [(labels[k], w) for k, w in wrongs.items()]


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _net(lib, cls, setting, prec, P, dev, **kw):
    net = getattr(lib, cls)(precision=prec, **setting, **kw)
    net.load_state_dict(P, strict=True)
    return net.to(dev)


def _score_net(lib, c, prec, P, dev):
    a = c["arch"]
    if a == "unet":
        return _net(lib, "ConditionalUNet", c["nets"][0][1], prec, P, dev)
    if a == "dunet":
        return _net(lib, "DenoisingUNet", c["nets"][0][1], prec, P, dev)
    if a == "dnafnet":
        return _net(lib, "DenoisingNAFNet", NAF3[1], prec, P, dev)
    if a == "nafnet":
        return _net(lib, "ConditionalNAFNet", NAF3[1], prec, P, dev)
    return _net(lib, "ConditionalNAFNet", NAF8[1], prec, P, dev, latent=True)


STEPS = {  # mode: (native mode name, the oracle's step as f(schedule, x, mu, noise, z, t), uses z)
    "sde": ("MODE_SDE", O.irsde_sde_step, True),
    "posterior": ("MODE_POSTERIOR", O.irsde_posterior_step, True),
    "dsde_sde": ("MODE_DSDE_SDE", lambda s, x, mu, e, z, t: O.dsde_sde_step(s, x, e, z, t), True),
    "dsde_ode": ("MODE_DSDE_ODE", lambda s, x, mu, e, z, t: O.dsde_ode_step(s, x, e, t), False),
}


def _step_check(lib, c, net, score, dev):
    """Teacher-forced sampler steps of every sde and mode of the case at each t:
    [(label, ratio to the bound, [(wrong label, ratio)])]."""
    mu, z = score["mu"], score["z"]
    d = lambda a: None if a is None else a.double()
    rows = []
    for kind, ms, T, modes in c["sdes"]:
        sc = _schedule(kind, ms, T)
        sde = (lib.IRSDE(ms, T, schedule="cosine", eps=0.005, device=dev) if kind == "irsde"
               else lib.DenoisingSDE(ms, T, device=dev))
        sde.set_model(net)
        for mode in modes:
            native, fn, uses_z = STEPS[mode]
            for k, t in enumerate(c["ts"]):
                x = score["calls"][k][2]
                eps = score["refs"][k].float()
                got = sde._native_step(getattr(lib._lib, native), x, mu, eps, z if uses_z else None, t).double()
                ref = fn(sc, x.double(), d(mu), eps.double(), d(z), t)
                err32 = (fn(sc, x, mu, eps, z, t).double() - ref).abs().max().item()
                lim = STEP_BOUND * max(err32, U * ref.abs().max().item())
                r = lambda a: (got - a).abs().max().item() / lim
                t2 = t + 1 if t == 1 else t - 1
                wrong = [("t=%d coefficients" % t2, r(fn(sc, x.double(), d(mu), eps.double(), d(z), t2)))]
                # the posterior's std at t = 1 is sqrt(1e-20 dt) * max_sigma: z has no effect there
                if uses_z and c["B"] > 1 and not (mode == "posterior" and t == 1):
                    wrong.append(("z rolled by one image", r(fn(sc, x.double(), d(mu), eps.double(),
                                                                torch.roll(z, 1, 0).double(), t))))
                rows.append(("%s %s(%s, %d) t=%d" % (mode, kind, ms, T, t), r(ref), wrong))
    return rows


def _pad_of(c, part, shape):
    s = _pad_step(c, part)[0]
    return (-shape[2]) % s, (-shape[3]) % s


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_task_network_vs_fp64_oracle(lib, case, prec, budget, capsys):
    c = case
    dev = _dev()
    refs = _oracle_refs(c, dev)
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    P = _weights(c)
    results, wrong, nets = [], [], []
    if c["arch"] == "latent":
        P, Pn = P
        ae = _net(lib, "UNet", AE[1], prec, P, dev)
        nets.append(ae)
        enc, dec = refs["encode"], refs["decode"]
        z, h = ae.encode(enc["img"])
        out = ae.decode(enc["ref"].float(), h)
        torch.cuda.synchronize()
        for part, got, r in (("encode", z, enc), ("decode", out, dec)):
            key = "%s %s" % (c["key"], part)
            pad = (0, 0) if part == "encode" else _pad_of(c, "encode", out.shape)
            results.append((key, part, _stats(got, r["ref"], pad)))
            wrong += [(key, label, _stats(got, w, pad)) for label, w in _wrong_refs(r["ref"], r["wrongs"])]
        P = Pn
    score = refs["score"]
    net = _score_net(lib, c, prec, P, dev)
    nets.append(net)
    key = c["key"] + (" nafnet" if c["arch"] == "latent" else "")
    mu = score["mu"]
    cond = c["arch"] in ("unet", "nafnet", "latent")
    gots = [net(x, mu, ts[0] if len(set(ts)) == 1 else ts) if cond else net(x, ts[0] if len(set(ts)) == 1 else ts)
            for _, ts, x in score["calls"]]
    torch.cuda.synchronize()
    pad = _pad_of(c, "score", gots[0].shape)
    k = c["ts"].index(c["tpm"])
    results += [(key, label, _stats(got, ref, pad)) for (label, _, _), got, ref in zip(score["calls"], gots, score["refs"])]
    wrong += [(key, label, _stats(gots[k], w, pad)) for label, w in _wrong_refs(score["refs"][k], score["wrongs"])]
    steps = _step_check(lib, c, net, score, dev)
    torch.cuda.synchronize()
    lib_bytes = sum(int(n._ctx.L.irsde_device_bytes(n._ctx.h)) for n in nets)
    peak = max(refs["peak"], torch.cuda.max_memory_reserved() + lib_bytes)
    seconds = time.perf_counter() - t0
    for n in nets:
        n._ctx.close()
    del nets, net
    band = lambda s: "  band %5.2f" % s["band"] if s["band"] is not None else ""
    with capsys.disabled():
        print("\n  %s (%s) %s: peak %s (library %s), oracle %.1f s, network %.1f s" % (
            c["id"], ", ".join(c["ymls"]), prec, _gb(peak), _gb(lib_bytes), refs["seconds"], seconds))
        for key, label, s in results:
            print("    %-24s %-18s max %.3e  rms %.3e  cell ratio %6.2f%s  -> %.3f of the bound" % (
                key, label, s["max"], s["rms"], s["cell"], band(s), _ratio(key, prec, s)))
        for key, label, s in wrong:
            print("    %-24s wrong reference: %-40s %.3g x the bound%s" % (key, label, _ratio(key, prec, s), band(s)))
        for label, r, w in steps:
            print("    step %-34s %.3f of the bound; wrong: %s" % (label, r, ", ".join("%s %.3g" % kv for kv in w)))
    for key, label, s in wrong:
        assert _ratio(key, prec, s) > 1.0, ("the bound does not see a wrong reference", key, label, s)
    for label, r, w in steps:
        for wl, rw in w:
            assert rw > 1.0, ("the step bound does not see a wrong reference", label, wl, rw)
    assert peak <= c["need"], (peak, c["need"])
    for key, label, s in results:
        assert _ratio(key, prec, s) <= 1.0, (key, label, s)
    for label, r, _ in steps:
        assert r <= 1.0, ("step", label, r)
