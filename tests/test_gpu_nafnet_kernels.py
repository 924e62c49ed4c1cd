"""Every kernel of nafnet.cu and elementwise.cu against a plain high-precision reference, through the standalone entries
irsde_nafnet_op, irsde_time_embedding, irsde_step_philox and irsde_prep_input: the same launchers the launch plan calls, on
pitched views, at the sizes where the kernels change code (16- vs 64-pixel pooling chunks at N = 1024 / 1025, the fused vs
two-pass SCA scaling, a 1-pixel last chunk, channel counts that are not a multiple of 8 or of a 64-channel block) and at a
2048x2048 level, whose 65536 pooling chunks do not fit in gridDim.y.

- NAFBlock ops (DenoisingNAFNet_arch.py:9-12,29-33,65-67,172-174): the depthwise 3x3 + SimpleGate + SCA chain against an fp64
  reference whose bound scales with fp64 sums of |terms|; SimpleGate, PixelShuffle + skip and the add bit for bit against
  the same torch ops in the storage type.  Every case also checks that nothing outside the written slices changes, that image
  1 of a batch of 3 equals the same image run alone and that two runs agree, bit for bit.
- Time embeddings (module_util.py:29-41, DenoisingUNet_arch.py:42-47, DenoisingNAFNet_arch.py:18-20,51-54) of both network
  families and the per-block table, against fp64 modules that follow oracle/irsde_oracle.py.
- The in-kernel Philox4x32-10 normals, against a numpy Philox with the kernel's counter layout (pinned to the Random123
  known-answer vectors without a GPU): x_T, single sampler steps, and a whole irsde_reverse(z = NULL) chain.
- The input packing (DenoisingUNet_arch.py:78-94, DenoisingNAFNet_arch.py:183-188) bit for bit against F.pad + cat.

Before a kernel is compared, each case proves that its bound rejects a set of wrong references (a pixel dropped from the
pool, a wrapping tap, a transposed SCA weight, another image's SCA, t +- 1, swapped sin / cos halves, another Philox stream,
block, uid or seed, ...).

test_every_compiled_kernel_has_a_case runs without a GPU: it compiles nafnet.cu and elementwise.cu and fails when an object
holds a kernel that neither a case below nor the table of kernels covered by other test files names.
"""
import ast
import ctypes
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24  # fp32 unit roundoff
DWGATE_SCA, SIMPLE_GATE, PIXEL_SHUFFLE_ADD, ADD = 0, 1, 2, 3
MODE_SDE, MODE_POSTERIOR, MODE_DSDE_SDE = 0, 2, 3
SEED = 0x9E3779B97F4A7C15  # both 32-bit halves non-zero
NOISE_STREAM = 0xFFFFFFFF  # the stream x_T is drawn from


def _tname(prec):
    return "float" if prec == "fp32" else "bf16"


# ------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------
def _dw(prec, H, W, c, B=3):
    N = H * W
    pix = 16 if N <= 1024 else 64
    nch = -(-N // pix)
    fused = N <= 1024
    T = _tname(prec)
    kernels = ["dwgate_kernel<%s>" % T, "sca_kernel<%s>" % T] + ([] if fused else ["scale_channels_kernel<%s>" % T])
    return dict(name="%s DWGATE_SCA %dx%d c=%d B=%d" % (prec, H, W, c, B), prec=prec, H=H, W=W, c=c, B=B, pix=pix, nch=nch,
                kernels=kernels, info=(pix, nch, 1 if fused else 2, 0))


DW_CASES = [_dw(p, H, W, c) for p in ("fp32", "bf16") for (H, W) in ((1, 1), (10, 12), (32, 32), (25, 41), (128, 128))
            for c in (6, 72, 512)] + [_dw(p, 2048, 2048, 8, B=1) for p in ("fp32", "bf16")]


def _ew(prec, kind, H, W, c):
    T = _tname(prec)
    kern = {SIMPLE_GATE: "simple_gate_kernel", PIXEL_SHUFFLE_ADD: "pixel_shuffle_add_kernel", ADD: "add_kernel"}[kind]
    label = {SIMPLE_GATE: "SIMPLE_GATE", PIXEL_SHUFFLE_ADD: "PIXEL_SHUFFLE_ADD", ADD: "ADD"}[kind]
    return dict(name="%s %s %dx%d c=%d" % (prec, label, H, W, c), prec=prec, kind=kind, H=H, W=W, c=c, B=3,
                kernels=["%s<%s>" % (kern, T)])


EW_CASES = [_ew(p, k, H, W, c) for p in ("fp32", "bf16") for (k, H, W, c) in
            ((SIMPLE_GATE, 7, 9, 5), (SIMPLE_GATE, 16, 16, 72), (PIXEL_SHUFFLE_ADD, 5, 7, 5), (PIXEL_SHUFFLE_ADD, 8, 8, 64),
             (ADD, 7, 9, 5), (ADD, 16, 16, 64))]

TIMES7 = [0.0, 1.0, 37.5, 100.0, 400.0, 4096.0, 7.0]


def _te(family, width, times):
    kernels = (["time_mlp_kernel"] if family == 0 else ["naf_time_mlp_kernel"]) + ["time_table_kernel"]
    return dict(name="%s width=%d rows=%d" % (["unet", "nafnet"][family], width, len(times)), family=family, width=width,
                times=times, S=3 * width + 5, kernels=kernels)


TE_CASES = [_te(f, w, ts) for f in (0, 1) for w in (4, 6, 64) for ts in ([1.0], TIMES7)]


def _prep(prec, H, W, Hp, Wp, C, pitch, cond, zero, border=False, B=2):
    name = "%s %dx%d->%dx%d C=%d pitch=%d %s %s%s" % (prec, H, W, Hp, Wp, C, pitch, "cond" if cond else "plain",
                                                    "zero" if zero else "reflect", " stem border" if border else "")
    return dict(name=name, prec=prec, B=B, C=C, H=H, W=W, Hp=Hp, Wp=Wp, pitch=pitch, cond=cond, zero=zero,
                pad=(3, 3, Wp + 8, Hp + 6) if border else (0, 0, 0, 0), kernels=["prep_input_kernel<%s>" % _tname(prec)])


PREP_CASES = [c for p in ("fp32", "bf16") for c in (
    _prep(p, 8, 6, 15, 11, 3, 6, 1, 0),                      # reflect at pad = H - 1 and W - 1
    _prep(p, 18, 23, 20, 24, 3, 6, 1, 1),                    # the NAFNet zero pad
    _prep(p, 9, 7, 12, 8, 3, 3, 0, 0),                       # not conditional
    _prep(p, 9, 7, 12, 8, 3, 8, 1, 0),                       # pitch above 2C: channels 6, 7 come back zero
    _prep(p, 20, 28, 24, 32, 3, 8, 1, 0, border=True),       # the tensor-core stem's zero-bordered buffer
)]

PHILOX_KERNELS = ["noise_state_kernel", "sde_update_kernel", "set_step_kernel", "advance_step_kernel"]

# kernels that the cases here do not reach, and the test function that checks each
COVERED_ELSEWHERE = {
    "nchw_to_nhwc_kernel<float>": ("test_gpu_conv_epilogues.py", "test_fused_conv_vs_fp64"),
    "nchw_to_nhwc_kernel<bf16>": ("test_gpu_conv_epilogues.py", "test_fused_conv_vs_fp64"),
    "nhwc_to_nchw_kernel<float>": ("test_gpu_conv_epilogues.py", "test_fused_conv_vs_fp64"),
    "nhwc_to_nchw_kernel<bf16>": ("test_gpu_conv_epilogues.py", "test_fused_conv_vs_fp64"),
    "s2d_kernel<float>": ("test_gpu_conv_epilogues.py", "test_fused_conv_vs_fp64"),
    "s2d_kernel<bf16>": ("test_gpu_conv_epilogues.py", "test_fused_conv_vs_fp64"),
    "split_tf32_kernel": ("test_gpu_conv_epilogues.py", "test_fused_conv_vs_fp64"),
    "sde_update_kernel": ("test_gpu_parity.py", "test_sde_steps_bitexact"),  # with z given and host t
    "random_states_kernel": ("test_gpu_parity.py", "test_generate_random_states_bit_exact"),
}


# ------------------------------------------------------------------------------------------------------------------
# (CPU) the cases name exactly the kernels the objects hold
# ------------------------------------------------------------------------------------------------------------------
def _normalize(demangled):
    m = re.search(r"irsde::(\w+(?:<[^>]*>)?)", demangled)
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
    compiled = {}
    for src in ("nafnet.cu", "elementwise.cu"):
        obj = str(tmp_path / (src + ".o"))
        r = subprocess.run([nvcc] + b.FLAGS + ["-c", os.path.join(b.CSRC, src), "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        s = subprocess.run([cuobjdump, "-res-usage", obj], capture_output=True, text=True, check=True)
        mangled = re.findall(r"Function (\S+?):", s.stdout)
        dem = subprocess.run([cufilt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.split("\n")
        compiled[src] = {_normalize(d) for d in dem if d.strip()}
    assert len(compiled["nafnet.cu"]) == 13, sorted(compiled["nafnet.cu"])
    assert len(compiled["elementwise.cu"]) == 16, sorted(compiled["elementwise.cu"])
    named = {k for c in DW_CASES + EW_CASES + TE_CASES + PREP_CASES for k in c["kernels"]} | set(PHILOX_KERNELS)
    named |= set(COVERED_ELSEWHERE)
    allk = compiled["nafnet.cu"] | compiled["elementwise.cu"]
    assert allk == named, ("without a case", sorted(allk - named), "not compiled", sorted(named - allk))


# ------------------------------------------------------------------------------------------------------------------
# numpy Philox4x32-10 with the kernel's counter layout (elementwise.cu normal4 / image_normals)
# ------------------------------------------------------------------------------------------------------------------
M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 arrays of uint32 values, key: 2 (arrays of) uint32 values -> 4 uint32 arrays."""
    c0, c1, c2, c3 = [np.asarray(v, dtype=np.uint64) & M32 for v in ctr]
    k0, k1 = [np.asarray(v, dtype=np.uint64) & M32 for v in key]
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return [v.astype(np.uint32) for v in (c0, c1, c2, c3)]


def test_philox_known_answers():
    """The generator above is Philox4x32-10: the Random123 known-answer vectors."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kat:
        got = tuple(int(v[0]) for v in philox4x32_10([[v] for v in ctr], key))
        assert got == want, ["%08x" % v for v in got]


def philox_normals(seed, uids, image_elems, stream, swap_uid=False, swap_seed=False, swap_cs=False, blk_add=0, blocks=None):
    """z [len(uids), image_elems] (fp64) as the kernel draws it: element j of the image with uid u is lane j % 4 of Philox
    block j // 4 with counter (block, uid lo, stream, 0x1234567 ^ uid hi) and key (seed lo, seed hi); the uniforms are
    formed in fp32 like normal4 forms them, Box-Muller in fp64 on them.  The keywords build the wrong generators.
    blocks = (b0, b1): only the elements 4 b0 .. 4 b1 - 1 of each image, [len(uids), 4 (b1 - b0)]."""
    b0, b1 = blocks if blocks is not None else (0, (image_elems + 3) // 4)
    nb = b1 - b0
    u = np.repeat(np.asarray([int(v) for v in uids], dtype=np.uint64), nb)
    blk = (np.tile(np.arange(b0, b1, dtype=np.int64), len(uids)) + blk_add) & 0xFFFFFFFF
    lo, hi = u & M32, u >> np.uint64(32)
    if swap_uid:
        lo, hi = hi, lo
    k = (seed & 0xFFFFFFFF, seed >> 32)
    if swap_seed:
        k = k[::-1]
    c = philox4x32_10([blk, lo, np.full(blk.shape, stream, dtype=np.uint64), np.uint64(0x1234567) ^ hi], k)
    two_m32 = np.float32(2.3283064365386963e-10)
    uf = [(v.astype(np.float32) + np.float32(0.5)) * two_m32 for v in c]
    u0 = np.minimum(np.maximum(uf[0], np.float32(1e-12)), np.float32(1.0)).astype(np.float64)
    u2 = np.minimum(np.maximum(uf[2], np.float32(1e-12)), np.float32(1.0)).astype(np.float64)
    a1 = (np.float32(6.283185307179586) * uf[1]).astype(np.float64)
    a3 = (np.float32(6.283185307179586) * uf[3]).astype(np.float64)
    r0, r1 = np.sqrt(-2.0 * np.log(u0)), np.sqrt(-2.0 * np.log(u2))
    cs, sn = (np.sin, np.cos) if swap_cs else (np.cos, np.sin)
    z = np.stack([r0 * cs(a1), r0 * sn(a1), r1 * cs(a3), r1 * sn(a3)], axis=-1)
    return z.reshape(len(uids), nb * 4)[:, :image_elems]


def _philox_mutations(t=None):
    m = [("uid halves swapped", dict(swap_uid=True)), ("seed halves swapped", dict(swap_seed=True)),
         ("cos / sin swapped", dict(swap_cs=True)), ("Philox block + 1", dict(blk_add=1)),
         ("Philox block - 1", dict(blk_add=-1))]
    if t is None:
        m.append(("stream 0 instead of x_T's", dict(stream=0)))
    else:
        m += [("stream t + 1", dict(stream=t + 1)), ("stream t - 1", dict(stream=t - 1)),
              ("x_T's stream reused", dict(stream=NOISE_STREAM))]
    return m


# ------------------------------------------------------------------------------------------------------------------
# GPU fixtures and helpers
# ------------------------------------------------------------------------------------------------------------------
def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
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


def _prec(c):
    return 1 if c["prec"] == "bf16" else 0


def _round(c, t):
    """The value the engine stores: bf16-rounded for precision 1."""
    return t.bfloat16().float() if c["prec"] == "bf16" else t


def _gen(c, dev):
    return torch.Generator(device=dev).manual_seed(sum(map(ord, c["name"])))


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _worst(err, bound):
    return (err.abs() / bound).max().item()


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same_outside(got, before, cols):
    """got / before: [rows, pitch] fp32; cols = (off, width) of the written slice: the rest must be bit-identical."""
    outside = torch.ones(got.shape[1], dtype=torch.bool, device=got.device)
    outside[cols[0]:cols[0] + cols[1]] = False
    return torch.equal(_bits(got[:, outside]), _bits(before[:, outside]))


def _naf_run(lib, ctx, c, kind, d, B=None, H=None, W=None, cc=None, prec=None, **over):
    """One irsde_nafnet_op call on copies of d's out / sca buffers; `over` replaces fields of the args struct."""
    a = lib._lib.NafArgs()
    out = d["out"].clone()
    sca = d["sca"].clone() if "sca" in d else None
    a.x, a.out = d["x"].data_ptr(), out.data_ptr()
    a.x_pitch, a.x_off = d["xv"]
    a.out_pitch, a.out_off = d["ov"]
    if "y" in d:
        a.y = d["y"].data_ptr()
        a.y_pitch, a.y_off = d["yv"]
    if kind == DWGATE_SCA:
        a.w, a.bias, a.sca_w, a.sca_b, a.sca = (d["w"].data_ptr(), d["bias"].data_ptr(), d["sw"].data_ptr(),
                                                d["sb"].data_ptr(), sca.data_ptr())
    for k, v in over.items():
        setattr(a, k, v)
    info = (ctypes.c_int32 * 4)()
    rc = ctx.L.irsde_nafnet_op(ctx.h, _prec(c) if prec is None else prec, kind, ctypes.byref(a), c["B"] if B is None else B,
                               c["H"] if H is None else H, c["W"] if W is None else W, c["c"] if cc is None else cc, info,
                               _stream())
    lib._lib.check(rc, ctx.h)
    torch.cuda.synchronize()
    return out, sca, tuple(info)


def _image(d, b, n_in, n_out):
    """The operands of image b alone (rows of the [B*pixels][pitch] buffers)."""
    one = dict(d)
    one["x"] = d["x"][b * n_in:(b + 1) * n_in].clone()
    one["out"] = d["out"][b * n_out:(b + 1) * n_out].clone()
    if "y" in d:
        one["y"] = d["y"][b * n_out:(b + 1) * n_out].clone()
    if "sca" in d:
        one["sca"] = d["sca"][b * d["c"]:].clone()
    return one


def _check_batch_and_repeat(lib, ctx, c, kind, d, out, sca, n_in, n_out):
    """A second run is bit-identical, and image 1 of the batch equals the same image run alone."""
    out2, sca2, _ = _naf_run(lib, ctx, c, kind, d)
    assert torch.equal(_bits(out2), _bits(out)), "two runs differ"
    if sca is not None:
        assert torch.equal(_bits(sca2), _bits(sca)), "two runs differ (sca)"
    if c["B"] < 3:
        return
    one = _image(d, 1, n_in, n_out)
    out1, sca1, _ = _naf_run(lib, ctx, c, kind, one, B=1)
    assert torch.equal(_bits(out1), _bits(out[n_out:2 * n_out])), "image 1 differs from the same image run alone"
    if sca is not None:
        assert torch.equal(_bits(sca1[:c["c"]]), _bits(sca[c["c"]:2 * c["c"]])), "image 1's sca differs when run alone"


# ------------------------------------------------------------------------------------------------------------------
# depthwise 3x3 + SimpleGate + SCA
# ------------------------------------------------------------------------------------------------------------------
def _dw_data(c, dev):
    g = _gen(c, dev)
    B, H, W, C, N = c["B"], c["H"], c["W"], c["c"], c["H"] * c["W"]
    rnd = lambda *s: torch.randn(*s, generator=g, device=dev)
    d = dict(c=C, xv=(2 * C + 8, 5), ov=(C + 8, 3))
    x = rnd(B, N, d["xv"][0])
    # planted pixels: the image's last pixel and the last pixel before the last chunk get a gate far above the typical
    # one, so that dropping either from the pool shows in bf16 too
    d["plant"] = [N - 1] + ([(c["nch"] - 1) * c["pix"] - 1] if c["nch"] > 1 else [])
    x[:, d["plant"]] *= 20.0 if N <= 16384 else 200.0
    d["x"] = _round(c, x.view(B * N, -1))
    d["w"] = rnd(2 * C, 9) * 0.4
    d["bias"] = rnd(2 * C) * 0.1
    d["sw"] = rnd(C, C) / math.sqrt(C)
    d["sb"] = rnd(C) * (0.5 / math.sqrt(N))  # comparable to sca_w @ mean: the bias and each mean both show
    d["out"] = _round(c, rnd(B * N, d["ov"][0]))
    d["sca"] = rnd(B * C + 64)
    return d


def _dw_ref(c, d, drop=None, mean_over_chunks=False, wrap=False, x1x1=False, shift2=False, sca_t=False, no_bias=False,
            other_image=False, mag=False):
    """fp64 reference of out [B, N, C] (and sca [B, C]); the keywords build the wrong references.  mag=True also returns
    the bound of out and of sca."""
    B, H, W, C, N = c["B"], c["H"], c["W"], c["c"], c["H"] * c["W"]
    bf = c["prec"] == "bf16"
    xo = d["xv"][1]
    x = d["x"].view(B, N, -1)[..., xo:xo + 2 * C].double()
    w = d["w"].double()
    dev = x.device
    # depthwise 3x3, zero padding: taps index the flattened pixel sequence, masked by row (and by column unless `wrap`)
    flat = F.pad(x.permute(0, 2, 1), (W + 1, W + 1))  # [B, 2C, N + 2W + 2]
    hh = torch.arange(N, device=dev) // W
    ww = torch.arange(N, device=dev) % W
    acc = d["bias"].double()[None, :, None].expand(B, 2 * C, N).clone()
    mag_acc = d["bias"].double().abs()[None, :, None].expand(B, 2 * C, N).clone()
    for r in range(3):
        for s in range(3):
            ok = ((hh + r - 1 >= 0) & (hh + r - 1 < H)).double()
            if not wrap:
                ok = ok * ((ww + s - 1 >= 0) & (ww + s - 1 < W)).double()
            o = (r - 1) * W + (s - 1)
            tap = flat[..., W + 1 + o:W + 1 + o + N] * ok
            acc = acc + w[:, r * 3 + s][None, :, None] * tap
            mag_acc = mag_acc + (w[:, r * 3 + s][None, :, None] * tap).abs()
    acc, mag_acc = acc.permute(0, 2, 1), mag_acc.permute(0, 2, 1)  # [B, N, 2C]
    x1, x2 = acc[..., :C], acc[..., C:]
    if shift2:
        x2 = torch.roll(x2, -1, dims=2)
    if x1x1:
        x2 = x1
    gate = x1 * x2
    if mag:
        # the kernel's fp32 gate: 9 fma per half from the bias (<= 10 u of the |terms| sum each), then one product
        e1, e2 = 10 * U * mag_acc[..., :C], 10 * U * mag_acc[..., C:]
        e_g = e1 * x2.abs() + x1.abs() * e2 + e1 * e2 + U * gate.abs()
    if bf:
        g_ref = gate.float().bfloat16().double()  # the stored gate the kernel pools
        if mag:
            # the kernel's fp32 gate rounds to the same bf16 value unless it lies within e_g of a rounding tie
            e = 2 * (e_g + U * gate.abs())
            amb = (gate - e).float().bfloat16() != (gate + e).float().bfloat16()
            d_g = torch.where(amb, 2 ** -7 * gate.abs() * 1.01 + e_g, torch.zeros_like(gate))
    else:
        g_ref = gate
        if mag:
            d_g = e_g
    pooled = g_ref
    if drop is not None:
        keep = torch.ones(N, dtype=torch.bool, device=dev)
        keep[drop] = False
        pooled = g_ref[:, keep]
    mean = pooled.sum(1) / (c["nch"] * c["pix"] if mean_over_chunks else N)  # [B, C]
    sw, sb = d["sw"].double(), d["sb"].double()
    sca = mean @ (sw if sca_t else sw.t()) + (0.0 if no_bias else sb)
    if other_image:
        sca = torch.roll(sca, 1, dims=0)
    out = g_ref * sca[:, None, :]
    if not mag:
        return out, sca
    # pooling: fp32 lanes over <= pix/4 pixels, a 2-level tree per chunk, then a serial sum over the chunks (each add
    # rounds by u of the running partial sum) and the division by N
    pad = c["nch"] * c["pix"] - N
    chunks = F.pad(g_ref.permute(0, 2, 1), (0, pad)).view(B, C, c["nch"], c["pix"]).sum(3)  # [B, C, nch]
    run = chunks.cumsum(2).abs().sum(2)
    gabs = g_ref.abs().sum(1)
    e_m = (d_g.sum(1) + U * (c["pix"] // 4 + 2) * gabs + U * run) / N + U * mean.abs()
    e_s = e_m @ sw.abs().t() + U * (C / 32 + 8) * (mean.abs() @ sw.abs().t() + sb.abs())
    u_out = 2 ** -8 * 1.01 if bf else U
    gq = g_ref.abs() + d_g
    bound = 2 * (d_g * sca.abs()[:, None, :] + gq * e_s[:, None, :] + u_out * gq * (sca.abs() + e_s)[:, None, :]) + 1e-300
    return out, sca, bound, 2 * e_s + 1e-300


def _dw_mutations(c, d):
    B, W, N = c["B"], c["W"], c["H"] * c["W"]
    m = [("the image's last pixel dropped from the pool", dict(drop=N - 1))]
    if c["nch"] > 1:
        m.append(("the last pixel before the last chunk dropped", dict(drop=d["plant"][1])))
    if c["nch"] * c["pix"] != N:
        m.append(("mean over nchunks * chunk pixels", dict(mean_over_chunks=True)))
    if W > 1:
        m.append(("horizontal taps wrap into the neighbouring row", dict(wrap=True)))
    m += [("x1 * x1", dict(x1x1=True)), ("second half shifted one channel", dict(shift2=True)),
          ("sca weight transposed", dict(sca_t=True)), ("sca without its bias", dict(no_bias=True))]
    if B > 1:
        m.append(("another image's sca", dict(other_image=True)))
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("case", DW_CASES, ids=[c["name"] for c in DW_CASES])
def test_dwgate_sca_vs_fp64(lib, scratch_ctx, case, capsys):
    c = case
    d = _dw_data(c, _dev())
    B, C, N = c["B"], c["c"], c["H"] * c["W"]
    ref, sca_ref, bound, sca_bound = _dw_ref(c, d, mag=True)
    for label, kw in _dw_mutations(c, d):
        r = _worst(_dw_ref(c, d, **kw)[0] - ref, bound)
        assert r > 1.0, ("the bound does not see", label, r)
    out, sca, info = _naf_run(lib, scratch_ctx, c, DWGATE_SCA, d)
    oo = d["ov"][1]
    assert _same_outside(out, d["out"], (oo, C)), "write outside the gate slice"
    assert torch.equal(_bits(sca[B * C:]), _bits(d["sca"][B * C:])), "write past sca"
    r = _worst(out[:, oo:oo + C].view(B, N, C).double() - ref, bound)
    r_sca = _worst(sca[:B * C].view(B, C).double() - sca_ref, sca_bound)
    with capsys.disabled():
        print("\n  info %-16s worst err / bound: out %.3f sca %.3f  %s" % (info, r, r_sca, c["name"]), end="")
    assert info == c["info"], (info, c["info"])
    assert r <= 1.0 and r_sca <= 1.0, (c["name"], r, r_sca)
    _check_batch_and_repeat(lib, scratch_ctx, c, DWGATE_SCA, d, out, sca, N, N)


# ------------------------------------------------------------------------------------------------------------------
# SimpleGate, PixelShuffle + skip, add: bit for bit against torch in the storage type
# ------------------------------------------------------------------------------------------------------------------
def _ew_data(c, dev):
    g = _gen(c, dev)
    B, H, W, C, kind = c["B"], c["H"], c["W"], c["c"], c["kind"]
    rnd = lambda *s: torch.randn(*s, generator=g, device=dev)
    n_in = H * W
    n_out = 4 * n_in if kind == PIXEL_SHUFFLE_ADD else n_in
    xw = {SIMPLE_GATE: 2 * C, PIXEL_SHUFFLE_ADD: 4 * C, ADD: C}[kind]
    d = dict(c=C, xv=(xw + 7, 3), ov=(C + 5, 2), n_in=n_in, n_out=n_out)
    d["x"] = _round(c, rnd(B * n_in, d["xv"][0]))
    if kind != SIMPLE_GATE:
        d["yv"] = (C + 9, 4)  # the pitched skip / second operand
        d["y"] = _round(c, rnd(B * n_out, d["yv"][0]))
    d["out"] = _round(c, rnd(B * n_out, d["ov"][0]))
    return d


def _ew_ref(c, d):
    """The same op in torch, in the storage type: a product or sum of two bf16 values is exact in fp32, so the kernel's one
    rounding to bf16 is torch's one rounding."""
    B, H, W, C, kind = c["B"], c["H"], c["W"], c["c"], c["kind"]
    st = torch.bfloat16 if c["prec"] == "bf16" else torch.float32
    xo, x = d["xv"][1], d["x"].to(st)
    if kind == SIMPLE_GATE:
        return (x[:, xo:xo + C] * x[:, xo + C:xo + 2 * C]).float()
    yo, y = d["yv"][1], d["y"].to(st)
    if kind == ADD:
        return (x[:, xo:xo + C] + y[:, yo:yo + C]).float()
    inp = x[:, xo:xo + 4 * C].reshape(B, H, W, 4 * C).permute(0, 3, 1, 2)
    skip = y[:, yo:yo + C].reshape(B, 2 * H, 2 * W, C)
    return (F.pixel_shuffle(inp, 2).permute(0, 2, 3, 1) + skip).reshape(B * 4 * H * W, C).float()


@pytest.mark.gpu
@pytest.mark.parametrize("case", EW_CASES, ids=[c["name"] for c in EW_CASES])
def test_nafnet_elementwise_bit_exact(lib, scratch_ctx, case):
    c = case
    d = _ew_data(c, _dev())
    out, _, info = _naf_run(lib, scratch_ctx, c, c["kind"], d)
    oo = d["ov"][1]
    assert info == (0, 0, 0, 0), info
    assert _same_outside(out, d["out"], (oo, c["c"])), "write outside the output slice"
    ref = _ew_ref(c, d)
    assert not torch.equal(_bits(ref), _bits(d["out"][:, oo:oo + c["c"]]))
    assert torch.equal(_bits(out[:, oo:oo + c["c"]]), _bits(ref)), c["name"]
    _check_batch_and_repeat(lib, scratch_ctx, c, c["kind"], d, out, None, d["n_in"], d["n_out"])


# ------------------------------------------------------------------------------------------------------------------
# time embeddings
# ------------------------------------------------------------------------------------------------------------------
def _te_data(c, dev):
    g = _gen(c, dev)
    w = c["width"]
    rnd = lambda *s: torch.randn(*s, generator=g, device=dev)
    n1 = 4 * w if c["family"] == 0 else 8 * w
    td_out = 4 * w if c["family"] == 0 else 2 * w
    d = dict(times=torch.tensor(c["times"], device=dev), td_out=td_out)
    d["w1"] = rnd(n1, w) * (1.5 / math.sqrt(w))  # pre-activations of order 1-2, where erf- and tanh-GELU differ most
    d["b1"] = rnd(n1) * 0.3
    d["w2"] = rnd(4 * w, 4 * w) / math.sqrt(4 * w)
    d["b2"] = rnd(4 * w) * 0.3
    d["wall"] = rnd(c["S"], td_out) / math.sqrt(td_out)
    d["ball"] = rnd(c["S"]) * 0.1
    return d


def _te_run(lib, c, d, family=None, rows=None, width=None, S=None):
    R = len(c["times"])
    temb = torch.full((R, d["td_out"]), float("nan"), device=d["times"].device)
    table = torch.full((R, c["S"]), float("nan"), device=d["times"].device)
    rc = lib._lib.load().irsde_time_embedding(
        c["family"] if family is None else family, _ptr(d["times"]), R if rows is None else rows,
        c["width"] if width is None else width, _ptr(d["w1"]), _ptr(d["b1"]), _ptr(d["w2"]), _ptr(d["b2"]), _ptr(d["wall"]),
        _ptr(d["ball"]), c["S"] if S is None else S, _ptr(temb), _ptr(table), _stream())
    lib._lib.check(rc)
    torch.cuda.synchronize()
    return temb, table


def _serial_err(v, wt, b):
    """Rounding of out[o] = sum_k v[k] wt[o][k] accumulated serially in fp32 (fma), then + b[o]: each step rounds by u of
    its partial sum, so the error is u times the sum of |partial sums| (first order; the fp64 partial sums stand in for the
    fp32 ones)."""
    cs = (v[:, None, :] * wt.double()[None]).cumsum(-1)
    return U * (cs.abs().sum(-1) + (cs[..., -1] + b.double()).abs())


def _warp_err(v, wt, b):
    """The same for time_table_kernel's warp dot product: lane l sums k = l, l + 32, ... serially, then 5 shuffle levels
    (each within u of the sum of |lane sums|) and + b."""
    t = v[:, None, :] * wt.double()[None]
    t = F.pad(t, (0, (-t.shape[-1]) % 32)).unflatten(-1, (-1, 32))
    cs = t.cumsum(-2)
    lane = cs[..., -1, :]
    return U * (cs.abs().sum((-2, -1)) + 5 * lane.abs().sum(-1) + (lane.sum(-1) + b.double()).abs())


def _te_ref(c, d, dt=0.0, swap=False, denom_half=False, tanh_gelu=False, gate_adjacent=False, other_row=False, mag=False):
    """fp64 temb [rows][td] and table [rows][S] (oracle time_embedding / the NAFNet lines of nafnet_forward); mag=True
    also returns their bounds."""
    w = c["width"]
    half = w // 2
    t = d["times"].double() + dt
    if other_row:
        t = torch.roll(t, 1)
    i = torch.arange(half, dtype=torch.float64, device=t.device)
    e = math.log(10000) / (half if denom_half else half - 1)
    f = torch.exp(-i * e)
    a = t[:, None] * f[None, :]
    emb = torch.cat((a.cos(), a.sin()) if swap else (a.sin(), a.cos()), dim=-1)
    lin = lambda v, wt, b: v @ wt.double().t() + b.double()
    p1 = lin(emb, d["w1"], d["b1"])
    if c["family"] == 0:
        h = F.gelu(p1, approximate="tanh" if tanh_gelu else "none")
        o = lin(h, d["w2"], d["b2"])
        temb = F.silu(o)
    else:
        td = 4 * w
        g = p1[:, :td] * (p1[:, 1:td + 1] if gate_adjacent else p1[:, td:])
        tt = lin(g, d["w2"], d["b2"])
        temb = tt[:, :2 * w] * tt[:, 2 * w:]
    table = lin(temb, d["wall"], d["ball"])
    if not mag:
        return temb, table
    # the kernel's argument: e = logf(10000) / (half - 1) and f = expf(-i e) in fp32 (f within (1 + i e) 2^-22 relative,
    # exact for i = 0), a = t * f rounded once; sinf / cosf within 2 ulp
    dA = lambda v, wt: v @ wt.double().abs().t()
    rel_f = torch.where(i == 0, torch.zeros_like(i), (1 + i * e) * 2 ** -22)
    d_emb = t.abs()[:, None] * f[None, :] * rel_f[None, :] + U * a.abs() * (i > 0) + 2 ** -22
    d_emb = torch.cat((d_emb, d_emb), dim=-1)
    d_p1 = dA(d_emb, d["w1"]) + _serial_err(emb, d["w1"], d["b1"])
    if c["family"] == 0:
        d_h = 1.13 * d_p1 + 4 * U * p1.abs()
        d_o = dA(d_h, d["w2"]) + _serial_err(h, d["w2"], d["b2"])
        d_t = 1.1 * d_o + 4 * U * o.abs()
    else:
        da, db = d_p1[:, :td], d_p1[:, td:]
        d_g = da * p1[:, td:].abs() + p1[:, :td].abs() * db + da * db + U * g.abs()
        d_tt = dA(d_g, d["w2"]) + _serial_err(g, d["w2"], d["b2"])
        da, db = d_tt[:, :2 * w], d_tt[:, 2 * w:]
        d_t = da * tt[:, 2 * w:].abs() + tt[:, :2 * w].abs() * db + da * db + U * temb.abs()
    d_tab = dA(d_t, d["wall"]) + _warp_err(temb, d["wall"], d["ball"])
    return temb, table, 2 * d_t + 1e-300, 2 * d_tab + 1e-300


def _te_mutations(c):
    m = [("t + 1", dict(dt=1.0)), ("t - 1", dict(dt=-1.0)), ("sin / cos halves swapped", dict(swap=True)),
         ("denominator half instead of half - 1", dict(denom_half=True))]
    m.append(("tanh-GELU", dict(tanh_gelu=True)) if c["family"] == 0 else ("gate (k, k+1) instead of (k, k+td)",
                                                                           dict(gate_adjacent=True)))
    if len(c["times"]) > 1:
        m.append(("another row", dict(other_row=True)))
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("case", TE_CASES, ids=[c["name"] for c in TE_CASES])
def test_time_embedding_vs_fp64(lib, case, capsys):
    c = case
    d = _te_data(c, _dev())
    temb_ref, tab_ref, b_t, b_tab = _te_ref(c, d, mag=True)
    for label, kw in _te_mutations(c):
        mt, mtab = _te_ref(c, d, **kw)
        r = max(_worst(mt - temb_ref, b_t), _worst(mtab - tab_ref, b_tab))
        assert r > 1.0, ("the bound does not see", label, r)
    temb, table = _te_run(lib, c, d)
    r_t, r_tab = _worst(temb.double() - temb_ref, b_t), _worst(table.double() - tab_ref, b_tab)
    with capsys.disabled():
        print("\n  worst err / bound: temb %.3f table %.3f  %s" % (r_t, r_tab, c["name"]), end="")
    assert r_t <= 1.0 and r_tab <= 1.0, (c["name"], r_t, r_tab)
    temb2, table2 = _te_run(lib, c, d)
    assert torch.equal(_bits(temb2), _bits(temb)) and torch.equal(_bits(table2), _bits(table))
    if len(c["times"]) > 1:  # a row does not depend on the others
        one = dict(d, times=d["times"][4:5].clone())
        t1, tab1 = _te_run(lib, dict(c, times=c["times"][4:5]), one)
        assert torch.equal(_bits(t1[0]), _bits(temb[4])) and torch.equal(_bits(tab1[0]), _bits(table[4]))


# ------------------------------------------------------------------------------------------------------------------
# in-kernel Philox
# ------------------------------------------------------------------------------------------------------------------
def _set_uids(lib, ctx, uids_mode, B):
    """-> the uid of each image of the next batch."""
    if uids_mode == "explicit":
        uids = [(7 << 32) | 3, 1, 0x123456789]  # high halves non-zero, out of order
        lib._lib.check(ctx.L.irsde_set_image_uids(ctx.h, (ctypes.c_uint64 * B)(*uids), B, _stream()), ctx.h)
        return uids
    base = 5 if uids_mode == "base 5" else 0
    lib._lib.check(ctx.L.irsde_set_image_base(ctx.h, base), ctx.h)
    return [base + b for b in range(B)]


def _z(seed, uids, n, stream, dev, **kw):
    return torch.from_numpy(philox_normals(seed, uids, n, stream, **kw)).to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("image_elems", [4096, 189, 1])
@pytest.mark.parametrize("uids_mode", ["default", "base 5", "explicit"])
def test_noise_state_vs_numpy_philox(lib, image_elems, uids_mode):
    """x_T = mu + z max_sigma with z from the numpy Philox (stream 0xffffffff); 189 elements per image: 4-element groups
    straddle images, 1 element: a group spans three images."""
    dev = _dev()
    B = 3
    sde = lib.IRSDE(10, 5, eps=0.005, device=dev)
    ctx = sde._ctx_for(torch.zeros(1, device=dev))
    uids = _set_uids(lib, ctx, uids_mode, B)
    mu = torch.rand(B, image_elems, device=dev, generator=torch.Generator(device=dev).manual_seed(image_elems))
    out = torch.empty_like(mu)
    lib._lib.check(ctx.L.irsde_noise_state_images(ctx.h, _ptr(mu), _ptr(out), B, image_elems, SEED, _stream()), ctx.h)
    torch.cuda.synchronize()
    ms = float(sde.max_sigma)
    z = _z(SEED, uids, image_elems, NOISE_STREAM, dev)
    ref = mu.double() + z * ms
    bound = ms * 2 ** -19 * (1 + z.abs()) + 2 ** -23 * (mu.double().abs() + (z * ms).abs())
    for label, kw in _philox_mutations():
        stream = kw.pop("stream", NOISE_STREAM)
        r = _worst(mu.double() + _z(SEED, uids, image_elems, stream, dev, **kw) * ms - ref, bound)
        assert r > 1.0, ("the bound does not see", label, r)
    r = _worst(out.double() - ref, bound)
    assert r <= 1.0, r
    lib._lib.check(ctx.L.irsde_set_image_base(ctx.h, 0), ctx.h)


def _sampler(lib, mode, dev):
    return lib.DenoisingSDE(25, 5, device=dev) if mode == MODE_DSDE_SDE else lib.IRSDE(10, 5, eps=0.005, device=dev)


@pytest.mark.gpu
@pytest.mark.parametrize("image_elems", [189, 4096])
@pytest.mark.parametrize("mode", [MODE_SDE, MODE_POSTERIOR, MODE_DSDE_SDE], ids=["SDE", "POSTERIOR", "DSDE_SDE"])
def test_step_philox_vs_step_with_numpy_z(lib, mode, image_elems):
    """irsde_step_philox at t draws z from stream t: it equals irsde_step fed the numpy Philox's z, up to the rounding of
    z itself, and no other stream, block, uid or seed does."""
    dev = _dev()
    B, t = 3, 3
    sde = _sampler(lib, mode, dev)
    g = torch.Generator(device=dev).manual_seed(mode * 7 + image_elems)
    x = torch.rand(B, image_elems, device=dev, generator=g)
    noise = torch.randn(B, image_elems, device=dev, generator=g)
    mu = torch.rand(B, image_elems, device=dev, generator=g) if mode != MODE_DSDE_SDE else None
    ctx = sde._ctx_for(x)
    uids = _set_uids(lib, ctx, "base 5", B)

    def step(z):
        out = torch.empty_like(x)
        lib._lib.check(ctx.L.irsde_step(ctx.h, mode, _ptr(x), _ptr(mu), _ptr(noise), _ptr(z.float().contiguous()), t, _ptr(out),
                                        x.numel(), _stream()), ctx.h)
        torch.cuda.synchronize()
        return out.double()

    z = _z(SEED, uids, image_elems, t, dev)
    ref = step(z)
    k = (step(torch.ones_like(x)) - step(torch.zeros_like(x))).abs()  # |d out / d z| (with the rounding of both)
    bound = k * 2 ** -19 * (1 + z.abs()) + 2 ** -22 * ref.abs() + 1e-300
    for label, kw in _philox_mutations(t):
        stream = kw.pop("stream", t)
        r = _worst(step(_z(SEED, uids, image_elems, stream, dev, **kw)) - ref, bound)
        assert r > 1.0, ("the bound does not see", label, r)
    out = torch.empty_like(x)
    lib._lib.check(ctx.L.irsde_step_philox(ctx.h, mode, _ptr(x), _ptr(mu), _ptr(noise), t, _ptr(out), B, image_elems, SEED,
                                           _stream()), ctx.h)
    torch.cuda.synchronize()
    r = _worst(out.double() - ref, bound)
    assert r <= 1.0, r
    lib._lib.check(ctx.L.irsde_set_image_base(ctx.h, 0), ctx.h)


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [0, 1], ids=["eager", "graph"])
@pytest.mark.parametrize("H,W", [(12, 16), (9, 7)])
def test_reverse_chain_equals_forward_and_philox_steps(lib, H, W, use_graph):
    """irsde_reverse(z = NULL), T = 3 on a schedule of 5, equals the loop noise_fn(x, t) + irsde_step_philox(t) for
    t = 3, 2, 1 bit for bit: the chain's set_step / advance_step kernels hand the update kernel stream t and its uids."""
    dev = _dev()
    torch.manual_seed(0)
    net = lib.ConditionalUNet(3, 3, 8, depth=2).to(dev)
    sde = lib.IRSDE(10, 5, eps=0.005, device=dev)
    sde.set_model(net)
    B, C, T = 2, 3, 3
    g = torch.Generator(device=dev).manual_seed(H * W)
    mu = torch.rand(B, C, H, W, device=dev, generator=g)
    xT = mu + torch.randn(B, C, H, W, device=dev, generator=g) * sde.max_sigma
    ctx = sde._ctx_for(xT)
    lib._lib.check(ctx.L.irsde_set_image_base(ctx.h, 3), ctx.h)
    x0 = torch.empty_like(xT)
    lib._lib.check(ctx.L.irsde_reverse(ctx.h, MODE_SDE, _ptr(xT), _ptr(mu), None, _ptr(x0), B, H, W, T, SEED, use_graph,
                                       _stream()), ctx.h)
    x = xT.clone()
    for t in range(T, 0, -1):
        eps, nxt = torch.empty_like(x), torch.empty_like(x)
        lib._lib.check(ctx.L.irsde_noise_fn(ctx.h, _ptr(x), _ptr(mu), lib._lib.float_array([t]), 1, _ptr(eps), B, H, W,
                                            _stream()), ctx.h)
        lib._lib.check(ctx.L.irsde_step_philox(ctx.h, MODE_SDE, _ptr(x), _ptr(mu), _ptr(eps), t, _ptr(nxt), B, C * H * W, SEED,
                                               _stream()), ctx.h)
        x = nxt
    torch.cuda.synchronize()
    assert not torch.equal(x, xT)
    assert torch.equal(_bits(x0), _bits(x))
    lib._lib.check(ctx.L.irsde_set_image_base(ctx.h, 0), ctx.h)


# ------------------------------------------------------------------------------------------------------------------
# input packing
# ------------------------------------------------------------------------------------------------------------------
def _prep_run(lib, c, xt, cnd, out, **over):
    a = dict(B=c["B"], C=c["C"], H=c["H"], W=c["W"], Hp=c["Hp"], Wp=c["Wp"], pitch=c["pitch"], cond=c["cond"], zero=c["zero"],
             pad_top=c["pad"][0], pad_left=c["pad"][1], row_pix=c["pad"][2], img_rows=c["pad"][3], prec=_prec(c))
    a.update(over)
    out = out.clone()
    rc = lib._lib.load().irsde_prep_input(a["prec"], _ptr(xt), _ptr(cnd), _ptr(out), a["B"], a["C"], a["H"], a["W"], a["Hp"],
                                          a["Wp"], a["pitch"], a["cond"], a["zero"], a["pad_top"], a["pad_left"], a["row_pix"],
                                          a["img_rows"], _stream())
    lib._lib.check(rc)
    torch.cuda.synchronize()
    return out


def _prep_data(c, dev):
    g = _gen(c, dev)
    B, C, H, W = c["B"], c["C"], c["H"], c["W"]
    rows, pix = (c["pad"][3], c["pad"][2]) if c["pad"][2] else (c["Hp"], c["Wp"])
    xt = torch.randn(B, C, H, W, device=dev, generator=g)
    cond = torch.randn(B, C, H, W, device=dev, generator=g)
    out = _round(c, torch.randn(B, rows, pix, c["pitch"], device=dev, generator=g))
    return xt, cond, out


@pytest.mark.gpu
@pytest.mark.parametrize("case", PREP_CASES, ids=[c["name"] for c in PREP_CASES])
def test_prep_input_bit_exact(lib, case):
    """The packed input equals F.pad(cat(xt - cond, cond)) in the storage type, zero channels up to the pitch, bit for bit;
    the border around the padded image comes back untouched."""
    c = case
    xt, cond, before = _prep_data(c, _dev())
    got = _prep_run(lib, c, xt, cond if c["cond"] else None, before)
    x = torch.cat([xt - cond, cond], dim=1) if c["cond"] else xt
    x = F.pad(x, (0, c["Wp"] - c["W"], 0, c["Hp"] - c["H"]), mode="constant" if c["zero"] else "reflect")
    x = F.pad(x.permute(0, 2, 3, 1), (0, c["pitch"] - x.shape[1]))
    ref = before.clone()
    pt, pl = c["pad"][:2]
    ref[:, pt:pt + c["Hp"], pl:pl + c["Wp"]] = _round(c, x)
    assert torch.equal(_bits(got), _bits(ref)), c["name"]


# ------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_entries_refuse_bad_arguments(lib, scratch_ctx):
    """Host-side validation: every call below describes a view outside its pitch, an empty image or batch, a reflect pad
    that would read outside the image, a border that does not fit, a width whose time MLP or SCA needs more than 48 KB of
    shared memory or a step without noise, and must be refused before anything is launched.  Every buffer has a generous
    tail, so a check that let one of these through would still stay inside the allocations."""
    dev = _dev()
    L = lib._lib
    tail = lambda t: torch.cat([t.reshape(-1), torch.zeros(1 << 18, device=dev)])
    # ---- irsde_nafnet_op
    c = _dw("fp32", 10, 12, 6)
    d = _dw_data(c, dev)
    d.update(x=tail(d["x"]), out=tail(d["out"]))
    xp, op = d["xv"][0], d["ov"][0]
    bad = [dict(x_off=xp - 12 + 1), dict(x_off=-1), dict(out_off=op - 6 + 1), dict(out_pitch=5, out_off=0), dict(sca=None),
           dict(B=0), dict(H=0), dict(W=0), dict(cc=0), dict(cc=12289, prec=0)]
    for kw in bad:
        with pytest.raises(L.IrsdeError):
            _naf_run(lib, scratch_ctx, c, DWGATE_SCA, d, **kw)
    _naf_run(lib, scratch_ctx, c, DWGATE_SCA, d)  # the unmodified call is accepted
    for kind in (PIXEL_SHUFFLE_ADD, ADD):
        c = _ew("fp32", kind, 5, 7, 5)
        d = _ew_data(c, dev)
        d.update(x=tail(d["x"]), y=tail(d["y"]), out=tail(d["out"]))
        for kw in (dict(y_off=d["yv"][0] - 5 + 1), dict(y=None), dict(x_pitch=4 * 5 if kind == PIXEL_SHUFFLE_ADD else 5)):
            with pytest.raises(L.IrsdeError):
                _naf_run(lib, scratch_ctx, c, kind, d, **kw)
        _naf_run(lib, scratch_ctx, c, kind, d)
    # ---- irsde_time_embedding
    c = TE_CASES[3]
    d = _te_data(c, dev)
    for kw in (dict(rows=0), dict(width=3), dict(width=2), dict(S=0), dict(family=2), dict(family=0, width=2458),
               dict(family=1, width=946)):
        with pytest.raises(L.IrsdeError):
            _te_run(lib, c, d, **kw)
    for family, width in ((0, 2456), (1, 944)):  # the widest that fit: accepted and run
        cw = _te(family, width, [400.0])
        _te_run(lib, cw, _te_data(cw, dev))
    # ---- irsde_create / irsde_create_nafnet
    with pytest.raises(L.IrsdeError):
        L.Context(3, 3, 2458, 2, L.NET_CONDITIONAL, L.PREC_FP32, 0)
    L.Context(3, 3, 2456, 2, L.NET_CONDITIONAL, L.PREC_FP32, 0).close()
    for width, levels in ((946, 1), (64, 8)):  # time MLP > 48 KB; SCA of the 16384-channel level > 48 KB
        with pytest.raises(L.IrsdeError):
            lib.nafnet._NafContext(3, width, 1, [1] * levels, [1] * levels, False, L.PREC_FP32, 0)
    lib.nafnet._NafContext(3, 944, 1, [1], [1], False, L.PREC_FP32, 0).close()
    # ---- irsde_prep_input
    c = _prep("fp32", 8, 6, 15, 11, 3, 6, 1, 0)
    xt, cond, out = _prep_data(c, dev)
    out = tail(out)
    for kw in (dict(Hp=16), dict(Wp=12), dict(Hp=7), dict(pitch=5), dict(cond=0, pitch=2), dict(B=0), dict(C=0),
               dict(pad_top=1), dict(pad_top=1, pad_left=0, row_pix=11, img_rows=15), dict(row_pix=10, img_rows=15)):
        with pytest.raises(L.IrsdeError):
            _prep_run(lib, c, xt, cond, out, **kw)
    with pytest.raises(L.IrsdeError):  # conditional without cond
        _prep_run(lib, c, xt, None, out)
    _prep_run(lib, c, xt, cond, out, Hp=16, zero=1)  # a zero pad reads nothing outside the image
    # ---- irsde_step_philox
    sde = lib.IRSDE(10, 5, eps=0.005, device=dev)
    x = torch.rand(3, 64, device=dev)
    ctx = sde._ctx_for(x)
    o = torch.empty(3 * 64 + (1 << 16), device=dev)
    step = lambda mode=MODE_SDE, t=3, B=3, n=64, mu=x: L.check(ctx.L.irsde_step_philox(
        ctx.h, mode, _ptr(x), _ptr(mu), _ptr(x), t, _ptr(o), B, n, SEED, _stream()), ctx.h)
    for kw in (dict(mode=1), dict(mode=4), dict(t=0), dict(t=6), dict(B=0), dict(n=0), dict(mu=None)):
        with pytest.raises(L.IrsdeError):
            step(**kw)
    L.check(ctx.L.irsde_set_image_uids(ctx.h, (ctypes.c_uint64 * 2)(4, 9), 2, _stream()), ctx.h)
    with pytest.raises(L.IrsdeError):  # two uids for a batch of three
        step()
    L.check(ctx.L.irsde_set_image_base(ctx.h, 0), ctx.h)
    step()
