"""The kernels at the image sizes the networks run at (2048² and 4096² levels, N >= 4 M pixels, buffers past 2^31 bytes),
through the standalone entry points, against fp64 references computed on the GPU on windows where errors land: the first
and last pixel rows of the first and last image (the last pixel of the last image has the largest element offset), the
seams between conv tiles, and seeded random windows.  Reductions over a whole image (the SCA mean, the LinearAttention
context, the full-attention softmax) are checked in full against fp64 with bounds that grow with the reduction length, and
each bound first rejects wrong references (a dropped last chunk or image, 1/N of another level, an off-by-one tile row,
another image's time row) before the kernel's output is accepted.  Everything outside the written view must come back
bit-identical.

Every case states its device-memory budget (at most 24 GB, the plan cache's default) in its id, skips when that much is not
free, and frees everything before the next case.  Before anything runs, the host computes the largest element offset and
grid dimensions the case implies and asserts that they fit the types the kernels use (test_case_extents_fit_the_kernels,
no GPU needed).

The last tests refuse every shape limit (gridDim.y / z <= 65535, H * W <= 2^30) at plan build on each network family and
on the standalone entries, with tiny images and nothing launched, and check that the context works afterwards.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_conv_epilogues import _conv_acc, _epilogue, _over_bound
from test_gpu_nafnet_kernels import SEED, _philox_mutations, philox_normals

GB = 1 << 30
BUDGET = 24 * GB
U = 2.0 ** -24
INT_MAX, GRID_YZ, GRID_X = 2 ** 31 - 1, 65535, 2 ** 31 - 1
QSM, AFF, SILU, RES, GEN = 1, 2, 4, 8, 16  # conv_tc.cu EK_*
NUM_SMS = 132


def _gamma(n):
    return n * U / (1 - n * U)


def _gb(n):
    return "%.1f GB" % (n / GB)


# ------------------------------------------------------------------------------------------------------------------
# cases, with the device bytes each one holds at its peak
# ------------------------------------------------------------------------------------------------------------------
def _conv(name, expect, engine, B, Cin, H, W, Cout, K, up=False, bias=False, silu=False, ss=None, res=False, qsm=False,
          out_view=None, crop=None, stem=False):
    """A conv of the launch plan at a real level size.  expect = (BN, MODE, EKT), or None (SIMT engine / the stem, which
    irsde_conv2d_ex runs without reporting it); ss = None | "shared" | "image"; crop = (h, w) of the fp32 NCHW head."""
    s, p = (2, 1) if K == 4 else (1, (K - 1) // 2)
    u = 2 if up else 1
    Ho, Wo = (H * u + 2 * p - K) // s + 1, (W * u + 2 * p - K) // s + 1
    c = dict(kind="conv", name=name, expect=expect, engine=engine, B=B, Cin=Cin, H=H, W=W, Cout=Cout, K=K, up=up, bias=bias,
             silu=silu, ss=ss, t_row=1, mv=False, qsm=qsm, in_view=(Cin, 0), out_view=out_view or (Cout, 0),
             res_view=(Cout, 0) if res else None, crop=crop, stem=stem, Ho=Ho, Wo=Wo)
    e = 2 if engine == 1 else 4
    npi, npo = B * H * W, B * Ho * Wo
    if stem:
        need = npi * Cin * 4 + npo * Cout * 4 + B * (H + 6) * (W + 8) * 8 * 2 + npo * Cout * 2
    else:
        need = npi * Cin * 4 + (B * Cout * crop[0] * crop[1] * 4 if crop else npo * c["out_view"][0] * 4)
        need += npo * Cout * 4 if res else 0
        if engine == 1:
            need += npi * Cin * 2 * (2 if K == 4 else 1) + (0 if crop else npo * c["out_view"][0] * 2) + (npo * Cout * 2 if res else 0)
        if engine == 2:
            need += 2 * npi * Cin * 4 + (npi * Cin * 4 if K == 4 else 0)
    c["need"] = int(need * 1.05) + 256 * 2 ** 20
    c["id"] = "%s, %s" % (name, _gb(c["need"]))
    return c


CONV_CASES = [
    _conv("bf16 ROWS 3x3 64->64 at 4096^2, time row + SiLU + residual, into a 72-ch buffer", (64, 2, GEN), 1, 1, 64, 4096,
          4096, 64, 3, silu=True, ss="shared", res=True, out_view=(72, 8)),
    _conv("bf16 ROWS 3x3 64->64 at 2048^2 B=2, per-image rows + SiLU + residual", (64, 2, GEN), 1, 2, 64, 2048, 2048, 64, 3,
          silu=True, ss="image", res=True),
    _conv("bf16 ROWS 3x3 64->192 at 2048^2 B=2 (two N tiles, plain division by tiles_m), per-image rows + SiLU",
          (128, 2, AFF | SILU), 1, 2, 64, 2048, 2048, 192, 3, silu=True, ss="image"),
    _conv("bf16 per-tap 4x4/2 64->128 at 4096^2, bias", (128, 0, AFF), 1, 1, 64, 4096, 4096, 128, 4, bias=True),
    _conv("bf16 per-tap nearest x2 + 3x3 128->64 to 4096^2, bias", (64, 0, AFF), 1, 1, 128, 2048, 2048, 64, 3, up=True,
          bias=True),
    _conv("bf16 per-tap N-fastest 1x1 64->384 q-softmax at 2048^2", (128, 0, QSM), 1, 1, 64, 2048, 2048, 384, 1, qsm=True),
    _conv("bf16 ROWS 3x3 head 64->3 at 4096^2, fp32 NCHW cropped to 4093x4090", (32, 2, GEN), 1, 1, 64, 4096, 4096, 3, 3,
          bias=True, crop=(4093, 4090)),
    _conv("bf16 7x7 stem 6->64 at 4096^2 (irsde_conv2d_ex)", None, 1, 1, 6, 4096, 4096, 64, 7, bias=True, stem=True),
    _conv("fp32x3 3x3 64->64 at 4096^2, time row + SiLU", (64, 3, GEN), 2, 1, 64, 4096, 4096, 64, 3, silu=True, ss="shared"),
    _conv("fp32x3 3x3 64->64 at 2048^2 B=2, per-image rows + SiLU + residual", (64, 3, GEN), 2, 2, 64, 2048, 2048, 64, 3,
          silu=True, ss="image", res=True),
    _conv("fp32x3 4x4/2 64->128 at 4096^2, bias", (128, 3, GEN), 2, 1, 64, 4096, 4096, 128, 4, bias=True),
    _conv("fp32x3 nearest x2 + 3x3 128->64 to 2048^2, bias", (64, 3, GEN), 2, 1, 128, 1024, 1024, 64, 3, up=True, bias=True),
    _conv("fp32x3 3x3 head 64->3 at 4096^2, fp32 NCHW cropped to 4093x4090", (32, 3, GEN), 2, 1, 64, 4096, 4096, 3, 3,
          bias=True, crop=(4093, 4090)),
    _conv("SIMT 3x3 64->64 at 4096^2, time row + SiLU + residual", None, 0, 1, 64, 4096, 4096, 64, 3, silu=True,
          ss="shared", res=True),
    _conv("SIMT 3x3 64->64 at 2048^2 B=2, per-image rows + SiLU, into a 72-ch buffer", None, 0, 2, 64, 2048, 2048, 64, 3,
          silu=True, ss="image", out_view=(72, 8)),
    _conv("SIMT 4x4/2 64->128 at 4096^2, bias", None, 0, 1, 64, 4096, 4096, 128, 4, bias=True),
    _conv("SIMT nearest x2 + 3x3 128->64 to 4096^2, bias", None, 0, 1, 128, 2048, 2048, 64, 3, up=True, bias=True),
]


def _tile_geometry(c):
    """(BN, BW, BH, tiles_m, tiles_n, num_tiles, n_fast) of the tensor-core descriptor conv_tc.cu builds for the case."""
    B, Cout, K = c["B"], c["Cout"], c["K"]
    Ha, Wa = (c["H"] // 2, c["W"] // 2) if K == 4 else (c["H"], c["W"])
    nph = 4 if c["up"] else 1
    if c["engine"] == 1:
        BN = 256 if Cout >= 256 else 128 if Cout > 64 else 64 if Cout > 32 else 32
        if BN == 256 and Cout % 256 and Cout % 128 == 0:
            BN = 128
    else:
        BN = 128 if Cout > 64 else 64 if Cout > 32 else 32
    best = None
    for bw in (128, 64, 32, 16, 8):
        bh = 128 // bw
        cost = -(-Wa // bw) * bw * -(-Ha // bh) * bh
        if best is None or cost < best[0]:
            best = (cost, bw, bh)
    _, BW, BH = best
    if c["engine"] == 1 and K == 3 and not c["up"] and BN <= 128:  # ROWS
        BW, BH = (16, 8) if Wa >= 16 else (8, 16)
    tiles_m = -(-Wa // BW) * -(-Ha // BH) * B * nph
    tiles_n = -(-Cout // BN)
    a_bytes = B * Ha * Wa * c["in_view"][0] * 2
    n_fast = c["engine"] == 1 and K == 1 and tiles_n > 1 and a_bytes > 24 << 20
    return BN, BW, BH, tiles_m, tiles_n, tiles_m * tiles_n, n_fast


def _plain_division(c):
    """The tile-decode divisors tc_fill_magic leaves to plain division: those d > 1 with (num_tiles + 2) d >= 2^32."""
    BN, BW, BH, tiles_m, tiles_n, num_tiles, n_fast = _tile_geometry(c)
    Ha, Wa = (c["H"] // 2, c["W"] // 2) if c["K"] == 4 else (c["H"], c["W"])
    divs = dict(tiles_m=tiles_m, tiles_n=tiles_n, tilesW=-(-Wa // BW), tilesH=-(-Ha // BH), B=c["B"])
    return sorted(k for k, d in divs.items() if d > 1 and (num_tiles + 2) * d >= 2 ** 32)


def _ln(prec, C, kind, B=2, N=2048 * 2048):
    """kind: 0 scalar, 1 vec, 2 geo (irsde_layernorm info[0])."""
    e = 2 if prec == "bf16" else 4
    npix = B * N
    need = npix * (2 * C + C + 16) * 4 + (npix * (3 * C + 16) * e if prec == "bf16" else 0)
    c = dict(kind="ln", prec=prec, C=C, B=B, N=N, expect=kind, in_pitch=C + (C % 4 and 4 - C % 4), out_view=(C + 16, 8))
    c["need"] = int(need * 1.05) + 256 * 2 ** 20
    c["name"] = "LayerNorm %s C=%d B=%d N=%d, per-image time rows + residual" % (prec, C, B, N)
    c["id"] = "%s, %s" % (c["name"], _gb(c["need"]))
    return c


LN_CASES = [_ln("fp32", 64, 2), _ln("fp32", 96, 1), _ln("fp32", 30, 0), _ln("bf16", 64, 2), _ln("bf16", 96, 1)]


def _att(prec, full, N, B=1):
    e = 2 if prec == "bf16" else 4
    npix = B * N
    need = npix * (384 + 128) * 4 + (npix * (384 + 128) * e if prec == "bf16" else 0) + (0 if full else npix * 256 * 8)
    c = dict(kind="att", prec=prec, full=full, N=N, B=B)
    c["need"] = int(need * 1.05) + 512 * 2 ** 20
    c["name"] = "%s attention %s B=%d N=%d" % ("full" if full else "linear", prec, B, N)
    c["id"] = "%s, %s" % (c["name"], _gb(c["need"]))
    return c


# linear: the C = 256 level (1024^2) of a 4096^2 input; full: the bottom of the denoising UNet at 2048^2 (256^2 keys)
ATT_CASES = [_att("fp32", False, 1024 * 1024), _att("bf16", False, 1024 * 1024), _att("fp32", True, 65536),
             _att("bf16", True, 65536)]


def _naf(prec, op, H, W, c, B=1):
    e = 2 if prec == "bf16" else 4
    ps = op == "PIXEL_SHUFFLE_ADD"
    npi = B * H * W
    npo = 4 * npi if ps else npi
    xw = 4 * c if ps else c if op == "ADD" else 2 * c
    bufs = npi * xw + (npo * c if op in ("ADD", "PIXEL_SHUFFLE_ADD") else 0) + npo * (c + 8)
    need = bufs * 4 + (bufs * e if prec == "bf16" else 0) + (npo * c * 4 if op != "DWGATE_SCA" else 0)
    if op == "DWGATE_SCA":
        need += 256 * 4096 * 2 * c * 8 * 3  # fp64 slabs of the reference
    d = dict(kind="naf", prec=prec, op=op, H=H, W=W, c=c, B=B)
    d["need"] = int(need * 1.05) + 256 * 2 ** 20
    d["name"] = "%s %s %dx%d c=%d B=%d" % (op, prec, H, W, c, B)
    d["id"] = "%s, %s" % (d["name"], _gb(d["need"]))
    return d


def _block(C, B, N):
    npix = B * N
    # x, out, xn (fp32) and the bf16 LayerNorm while the entry holds its bf16 copies of x, out and xn; the fp64 slabs of the
    # reference come before out and xn exist
    need = npix * C * (4 * 3 + 2) + npix * C * 2 * 3
    c = dict(kind="block", C=C, B=B, N=N, need=int(need * 1.03) + 2 ** 29)
    c["name"] = "linattn block C=%d B=%d N=%d" % (C, B, N)
    c["id"] = "%s, %s" % (c["name"], _gb(c["need"]))
    return c


# level 0 of a 4096^2 input (C = 64) and the 2048^2 levels; C = 128 at 4096^2 needs 8.6 GB per buffer and does not fit
BLOCK_CASES = [_block(64, 1, 4096 * 4096), _block(64, 2, 2048 * 2048), _block(128, 2, 2048 * 2048)]

NAF_CASES = ([_naf(p, "DWGATE_SCA", 4096, 4096, 32) for p in ("fp32", "bf16")] +
             [_naf(p, op, 4096, 4096, 32) for p in ("fp32", "bf16") for op in ("SIMPLE_GATE", "ADD")] +
             [_naf(p, "PIXEL_SHUFFLE_ADD", 2048, 2048, 32) for p in ("fp32", "bf16")])

PREP = dict(kind="prep", B=16, C=3, H=4090, W=4093, Hp=4096, Wp=4096, pitch=8)
PREP["need"] = PREP["B"] * PREP["Hp"] * PREP["Wp"] * PREP["pitch"] * 4 + 2 * PREP["B"] * 3 * PREP["H"] * PREP["W"] * 4 + GB // 2
PHILOX = dict(kind="philox", B=43, E=3 * 4096 * 4096)  # 2.16e9 elements: x (updated in place) and noise
PHILOX["need"] = 2 * PHILOX["B"] * PHILOX["E"] * 4 + GB // 2
IMG = dict(kind="img", B=8, H=4096, W=4096, C=3)
IMG["need"] = 2 * IMG["B"] * IMG["H"] * IMG["W"] * 3 * 4 + 2 * IMG["B"] * IMG["H"] * IMG["W"] * 3 + GB // 2


# ------------------------------------------------------------------------------------------------------------------
# (CPU) the largest element offsets and grid dimensions each case implies fit the kernels' types
# ------------------------------------------------------------------------------------------------------------------
def _extents(c):
    """[(what, value, limit)]: offsets the kernels form in 64 bits, counts and indices they hold in int, grid dimensions."""
    k = c["kind"]
    I64 = 2 ** 63 - 1
    if k == "conv":
        B, H, W, Ho, Wo = c["B"], c["H"], c["W"], c["Ho"], c["Wo"]
        ex = [("largest input element offset", B * H * W * c["in_view"][0] - 1, I64),
              ("largest output element offset", B * Ho * Wo * c["out_view"][0] - 1, I64),
              ("pixels of one output image (int)", Ho * Wo, 2 ** 30),
              ("input / output rows, columns (int)", max(H, W, Ho, Wo) * 2, INT_MAX)]
        if c["engine"] == 0:
            ex += [("SIMT gridDim.x", -(-B * Ho * Wo // 64), GRID_X), ("SIMT gridDim.y", -(-c["Cout"] // 64), GRID_YZ)]
        elif not c["stem"]:
            num_tiles = _tile_geometry(c)[5]
            ex += [("num_tiles + gridDim.x (int tile loop)", num_tiles + NUM_SMS, INT_MAX)]
        return ex
    if k == "ln":
        npix = c["B"] * c["N"]
        return [("largest element offset", npix * (c["C"] + 8) - 1, 2 ** 63 - 1), ("N (int)", c["N"], INT_MAX),
                ("gridDim.x", npix, GRID_X)]
    if k == "att":
        B, N = c["B"], c["N"]
        return [("largest qkv element offset", B * N * 384 - 1, 2 ** 63 - 1), ("N (int)", N, 2 ** 30),
                ("gridDim.y", 4 * B if c["full"] else B, GRID_YZ), ("gridDim.x", -(-N // 64), GRID_X)]
    if k == "block":
        B, N, C = c["B"], c["N"], c["C"]
        return [("largest element offset", B * N * C - 1, 2 ** 63 - 1), ("N (int)", N, 2 ** 30), ("gridDim.y", B, GRID_YZ),
                ("chunk index (int)", -(-N // 64), INT_MAX)]
    if k == "naf":
        B, H, W, cc = c["B"], c["H"], c["W"], c["c"]
        n_out = B * H * W * (4 if c["op"] == "PIXEL_SHUFFLE_ADD" else 1)
        nchunks = -(-H * W // 64)
        return [("largest out element offset", n_out * (cc + 8) - 1, 2 ** 63 - 1), ("H * W (int)", H * W, 2 ** 30),
                ("elements / 256 (gridDim.x)", -(-n_out * cc // 256), GRID_X), ("dwgate gridDim.z", B, GRID_YZ),
                ("dwgate chunk index (int)", nchunks + GRID_YZ, INT_MAX)]
    if k == "prep":
        n = c["B"] * c["Hp"] * c["Wp"] * c["pitch"]
        return [("largest element offset", n - 1, 2 ** 63 - 1), ("elements (past 2^31)", 2 ** 31, n),
                ("gridDim.x", -(-c["B"] * c["Hp"] * c["Wp"] // 256), GRID_X)]
    if k == "philox":
        n = c["B"] * c["E"]
        return [("largest element offset", n - 1, 2 ** 63 - 1), ("elements (past 2^31)", 2 ** 31, n),
                ("gridDim.x", -(-n // 4 // 256), GRID_X)]
    if k == "img":
        B, H, W = c["B"], c["H"], c["W"]
        return [("largest fp32 element offset", B * 3 * H * W - 1, 2 ** 63 - 1), ("gridDim.y", B, GRID_YZ),
                ("tensor2img gridDim.x", -(-H * W // 1024), GRID_X), ("ssim tiles (int)", (H // 16 + 1) * (W // 16 + 1), INT_MAX)]
    raise AssertionError(k)


ALL_CASES = CONV_CASES + LN_CASES + ATT_CASES + BLOCK_CASES + NAF_CASES + [PREP, PHILOX, IMG]


def _check_extents(c):
    for what, v, lim in _extents(c):
        assert 0 <= v <= lim, (c.get("name", c["kind"]), what, v, lim)
    assert c["need"] <= BUDGET, (c.get("name", c["kind"]), c["need"])


@pytest.mark.parametrize("case", ALL_CASES, ids=[c.get("id", c["kind"]) for c in ALL_CASES])
def test_case_extents_fit_the_kernels(case):
    _check_extents(case)
    if case["kind"] == "conv" and case["engine"] != 0 and not case["stem"]:
        # the ROWS 4096^2 conv has 131072 M tiles: its tile decode divides by tiles_m with plain division
        if case["B"] * case["H"] * case["W"] == 4096 * 4096 and case["expect"][1] == 2:
            assert "tiles_m" in _plain_division(case)
        if case["Cout"] == 192:  # decoded with tile / tiles_m = 1 for the second N tile
            assert "tiles_m" in _plain_division(case) and _tile_geometry(case)[4] == 2


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
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


@pytest.fixture
def budget(request):
    """Checks the case's extents, skips unless its bytes are free, and frees everything the case allocated afterwards."""
    c = request.node.callspec.params.get("case") if hasattr(request.node, "callspec") else None
    _dev()
    torch.cuda.empty_cache()
    _check_extents(c)
    free, _ = torch.cuda.mem_get_info()
    if free < c["need"]:
        pytest.skip("needs %d bytes of device memory, %d free" % (c["need"], free))
    torch.cuda.reset_peak_memory_stats()
    yield c
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _bits(t):
    return t.contiguous().view(torch.int32)


def _lib_bytes(ctx):
    """Device bytes the library has allocated on ctx so far: the entries never give the count back when they free their
    scratch, so the growth over a case is what the library held on top of torch during it."""
    return ctx.L.irsde_device_bytes(ctx.h)


def _report(c, worst, wrong, extra="", lib_bytes=0):
    """Prints the worst error / bound, each wrong reference's ratio and the device memory the case held at its peak (torch's
    reserved peak + the library's scratch), and checks the ratios are all > 1 and the peak is within the budget."""
    peak = torch.cuda.max_memory_reserved() + lib_bytes
    print("\n  %-78s worst %.3f  wrong refs %s  peak %s (library %s) %s" % (
        c.get("name", c["kind"]), worst, " ".join("%s=%.3g" % kv for kv in wrong), _gb(peak), _gb(lib_bytes), extra), end="")
    for label, r in wrong:
        assert r > 1.0, ("the bound does not see a wrong reference", label, r)
    assert peak <= BUDGET, (c.get("name", c["kind"]), peak)


def _windows(n_rows, B, seam, seed, rows=2):
    """(image, r0, r1) output-row windows: first rows of image 0, last rows of the last image, a tile seam, random rows."""
    g = np.random.default_rng(seed)
    w = [(0, 0, rows), (B - 1, n_rows - rows, n_rows)]
    if seam and seam + rows // 2 < n_rows:
        w.append((0, seam - rows // 2, seam + rows // 2))
        mid = (n_rows // 2 // seam) * seam
        if mid >= rows // 2:
            w.append((B - 1, mid - rows // 2, mid + rows // 2))
    for _ in range(2):
        r0 = int(g.integers(0, n_rows - rows))
        w.append((int(g.integers(0, B)), r0, r0 + rows))
    return w


# ------------------------------------------------------------------------------------------------------------------
# GPU: convolutions
# ------------------------------------------------------------------------------------------------------------------
def _conv_data(c, dev):
    g = torch.Generator(device=dev).manual_seed(sum(map(ord, c["name"])))
    B, Cin, H, W, Cout, K, Ho, Wo = (c[k] for k in ("B", "Cin", "H", "W", "Cout", "K", "Ho", "Wo"))
    d = {}
    if c["stem"]:
        d["x"] = torch.randn(B, Cin, H, W, generator=g, device=dev)
    else:
        d["x"] = torch.randn(B, H, W, c["in_view"][0], generator=g, device=dev)
    if c["engine"] == 1:
        d["x"].copy_(d["x"].bfloat16())
    d["w"] = torch.randn(Cout, Cin, K, K, generator=g, device=dev) / (Cin * K * K) ** 0.5
    d["bias"] = 0.5 * torch.randn(Cout, generator=g, device=dev) if c["bias"] else None
    d["mv"] = None
    if c["ss"]:
        d["stride"] = 1 if c["ss"] == "image" else 0
        d["rows"] = c["t_row"] + (B - 1) * d["stride"] + 2
        d["ss_off"] = 16
        d["S"] = d["ss_off"] + 2 * Cout + 8
        d["ss"] = torch.rand(d["rows"], d["S"], generator=g, device=dev) * 2 - 1
    if c["res_view"]:
        d["res"] = torch.randn(B, Ho, Wo, Cout, generator=g, device=dev)
        d["res"].copy_(d["res"].bfloat16())
    if c["stem"]:
        d["y"] = torch.full((B, Cout, Ho, Wo), 7.0, device=dev)
    elif c["crop"]:
        d["y"] = torch.randn(B * Cout * c["crop"][0] * c["crop"][1] + 4096, generator=g, device=dev)
    else:
        d["y"] = torch.randn(B, Ho, Wo, c["out_view"][0], generator=g, device=dev)
        d["y"].copy_(d["y"].bfloat16())  # bf16 values: the bf16 engine's round trip keeps them exactly
    return d


def _conv_run(lib, ctx, c, d):
    s, p = (2, 1) if c["K"] == 4 else (1, (c["K"] - 1) // 2)
    info = (ctypes.c_int32 * 4)()
    if c["stem"]:
        rc = ctx.L.irsde_conv2d_ex(ctx.h, 1, _ptr(d["x"]), _ptr(d["w"]), _ptr(d["bias"]), None, _ptr(d["y"]), c["B"], c["Cin"],
                                   c["H"], c["W"], c["Cout"], 7, 7, 1, 3, 0, 0, 0, _stream())
    else:
        ptr = lambda t: t.data_ptr() if t is not None else None
        ep = lib._lib.ConvEpilogue()
        ep.bias, ep.res = ptr(d["bias"]), ptr(d.get("res"))
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
        rc = ctx.L.irsde_conv2d_fused(ctx.h, c["engine"], _ptr(d["x"]), _ptr(d["w"]), ctypes.byref(ep), _ptr(d["y"]), c["B"],
                                      c["Cin"], c["H"], c["W"], c["Cout"], c["K"], c["K"], s, p, int(c["up"]), info, _stream())
    lib._lib.check(rc, ctx.h)
    torch.cuda.synchronize()
    return tuple(info)


def _conv_window_acc(c, d, b, r0, r1, dtype):
    """The conv of image b, output rows r0..r1-1 (full width), NCHW in `dtype`: _conv_acc on the input rows those outputs
    read, plus a halo whose own outputs (which see the slab's zero border) are dropped."""
    K, H = c["K"], c["H"]
    if K == 4:
        a, e = max(0, 2 * r0 - 2), min(H, 2 * r1 + 2)
        lo = a // 2
    elif c["up"]:
        a, e = max(0, r0 // 2 - 1), min(H, (r1 + 1) // 2 + 1)
        lo = 2 * a
    else:
        h = K // 2
        a, e = max(0, r0 - h), min(H, r1 + h)
        lo = a
    if c["stem"]:
        x = d["x"][b:b + 1, :, a:e].to(dtype)
        w = d["w"].bfloat16().to(dtype)
        # zero rows only at the image's own borders: output j is image row a - top + j + 3
        top, bot = (3 if a == 0 else 0), (3 if e == H else 0)
        acc = F.conv2d(F.pad(x, (3, 3, top, bot)), w)
        lo = a + 3 - top
        return acc[:, :, r0 - lo:r1 - lo]
    slab = d["x"][b:b + 1, a:e]
    acc = _conv_acc(dict(c, B=1, H=e - a), dict(d, x=slab), dtype)
    return acc[:, :, r0 - lo:r1 - lo]


def _conv_window_ref(c, d, b, r0, r1, dtype=torch.float64, **mut):
    acc = _conv_window_acc(c, d, b, r0, r1, dtype)
    if c["stem"]:
        return acc + d["bias"].to(acc)[None, :, None, None]
    d2 = dict(d)
    if c["res_view"]:
        d2["res"] = d["res"][b:b + 1, r0:r1]
    rows = None
    if c["ss"]:
        rows = [mut.pop("rows", c["t_row"] + b * d["stride"])]
    return _epilogue(dict(c, B=1, crop=None), d2, acc, rows=rows, **mut)


def _conv_got(c, y, b, r0, r1):
    if c["stem"]:
        return y[b:b + 1, :, r0:r1].double()
    if c["crop"]:
        ch, cw = c["crop"]
        n = c["B"] * c["Cout"] * ch * cw
        return y[:n].view(c["B"], c["Cout"], ch, cw)[b:b + 1, :, r0:r1].double()
    off = c["out_view"][1]
    return y[b:b + 1, r0:r1, :, off:off + c["Cout"]].permute(0, 3, 1, 2).double()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CONV_CASES, ids=[c["id"] for c in CONV_CASES])
def test_conv_at_level_size_vs_fp64(lib, scratch_ctx, case, budget, capsys):
    c = case
    dev = _dev()
    d = _conv_data(c, dev)
    n_rows = c["crop"][0] if c["crop"] else c["Ho"]
    crop_w = c["crop"][1] if c["crop"] else None
    geo = None if (c["engine"] == 0 or c["stem"]) else _tile_geometry(c)
    seam = (geo[2] * (2 if c["up"] else 1)) if geo else 64
    wins = _windows(n_rows, c["B"], seam, len(c["name"]))
    # what the buffer held before the call: the windows, the channels outside the view, the guard band
    before = {w: _conv_got(c, d["y"], *w).clone() for w in wins}
    pitch, off = c["out_view"]
    outside = None
    if not c["crop"] and not c["stem"] and pitch > c["Cout"]:
        sel = torch.ones(pitch, dtype=torch.bool, device=dev)
        sel[off:off + c["Cout"]] = False
        outside = (sel, d["y"][..., sel].clone())
    guard = d["y"][-4096:].clone() if c["crop"] else None

    def ref_of(b, r0, r1, dtype=torch.float64, **mut):
        r = _conv_window_ref(c, d, b, r0, r1, dtype, **mut)
        return r[..., :crop_w] if crop_w else r

    def err32_of(b, r0, r1, ref):
        if c["engine"] != 2:
            return 0.0
        return (ref_of(b, r0, r1, torch.float32).double() - ref).abs().max().item()

    ratio = lambda got, ref, e32: _over_bound(dict(c, engine=1 if c["stem"] else c["engine"]), got, ref, e32)
    # wrong references: an off-by-one tile row, a dropped last image (its rows left as they were), another time row
    b, r0, r1 = wins[1]
    ref = ref_of(b, r0, r1)
    e32 = err32_of(b, r0, r1, ref)
    wrong = [("row-1", ratio(ref_of(b, r0 - 1, r1 - 1), ref, e32)), ("dropped last image", ratio(before[wins[1]], ref, e32))]
    if c["ss"]:
        t = c["t_row"] + b * d["stride"]
        wrong += [("time row+1", ratio(ref_of(b, r0, r1, rows=t + 1), ref, e32)),
                  ("scale/shift swapped", ratio(ref_of(b, r0, r1, swap_ss=True), ref, e32))]
    lb0 = _lib_bytes(scratch_ctx)
    info = _conv_run(lib, scratch_ctx, c, d)
    lib_bytes = _lib_bytes(scratch_ctx) - lb0
    worst = 0.0
    for w in wins:
        ref = ref_of(*w)
        got = _conv_got(c, d["y"], *w)
        assert got.shape == ref.shape, (got.shape, ref.shape)
        worst = max(worst, ratio(got, ref, err32_of(*w, ref)))
    extra = ""
    if geo:
        extra = "<%d,%d,%d> num_tiles %d (BW %d BH %d) plain division: %s" % (info[0], info[1], info[2], info[3], geo[1], geo[2],
                                                                            ",".join(_plain_division(c)) or "none")
    with capsys.disabled():
        _report(c, worst, wrong, extra, lib_bytes)
    if geo:
        assert info[:3] == c["expect"], (info, c["expect"])
        assert info[3] == geo[5], (info, geo)
    if outside is not None:
        assert torch.equal(_bits(d["y"][..., outside[0]]), _bits(outside[1])), "write outside the output view"
    if guard is not None:
        assert torch.equal(_bits(d["y"][-4096:]), _bits(guard)), "write past the cropped output"
    assert worst <= 1.0, worst


# ------------------------------------------------------------------------------------------------------------------
# GPU: LayerNorm
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", LN_CASES, ids=[c["id"] for c in LN_CASES])
def test_layernorm_at_4m_pixels_vs_fp64(lib, scratch_ctx, case, budget, capsys):
    c = case
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(c["C"] * 7 + len(c["prec"]))
    B, N, C = c["B"], c["N"], c["C"]
    bf = c["prec"] == "bf16"
    rnd = lambda t: t.bfloat16().float() if bf else t
    x = torch.randn(B * N, c["in_pitch"], generator=g, device=dev).add_(2.0)
    res = torch.randn(B * N, C, generator=g, device=dev)
    if bf:
        x.copy_(x.bfloat16())
        res.copy_(res.bfloat16())
    gain = 1 + 0.5 * torch.randn(C, generator=g, device=dev)
    S, t_row = 2 * C + 16, 1
    ss = torch.rand(B + 3, S, generator=g, device=dev) * 2 - 1
    pitch, off = c["out_view"]
    y = torch.randn(B * N, pitch, generator=g, device=dev)
    y.copy_(y.bfloat16())
    out_before = y[:, :off].clone(), y[:, off + C:].clone()
    wins = [(b, p0, p0 + 64) for b, p0 in ((0, 0), (B - 1, N - 64), (0, N // 2 - 32), (B - 1, 12345 * 64 + 17))]

    def ref_of(b, p0, p1, row=None, unbiased=False):
        xs = x[b * N + p0:b * N + p1, :C].double()
        mean = xs.mean(1, keepdim=True)
        var = xs.var(1, unbiased=unbiased, keepdim=True)
        xh = (xs - mean) / torch.sqrt(var + 1e-5) * gain.double()
        r = ss[t_row + b if row is None else row].double()
        core = xh * (r[8:8 + C] + 1)
        return core + r[8 + C:8 + 2 * C] + res[b * N + p0:b * N + p1].double(), core, (mean.abs() / var.sqrt())

    def bound_of(ref, core, rel):
        b = (C + 16) * U * 4 * (1 + rel) * core.abs() + 4 * U * (ref.abs() + core.abs() + 1)
        return (1 + 2 ** -8) * b + 2 ** -8 * ref.abs() if bf else b  # bf16 output: unit roundoff 2^-8 of the fp32 result

    b, p0, p1 = wins[1]
    ref, core, rel = ref_of(b, p0, p1)
    bound = bound_of(ref, core, rel)
    wrong = [("image 0's time row", ((ref_of(b, p0, p1, row=t_row)[0] - ref).abs() / bound).max().item()),
             ("dropped last image", ((y[b * N + p0:b * N + p1, off:off + C].double() - ref).abs() / bound).max().item())]
    if not bf:
        wrong.append(("unbiased variance", ((ref_of(b, p0, p1, unbiased=True)[0] - ref).abs() / bound).max().item()))
    a = lib._lib.LnArgs()
    a.g, a.res, a.ss = gain.data_ptr(), res.data_ptr(), ss.data_ptr()
    a.in_pitch, a.in_off, a.res_pitch, a.res_off, a.out_pitch, a.out_off = c["in_pitch"], 0, C, 0, pitch, off
    a.ss_rows, a.ss_S, a.off_scale, a.off_shift, a.ss_img_stride, a.t_row = B + 3, S, 8, 8 + C, 1, t_row
    info = (ctypes.c_int32 * 4)()
    lb0 = _lib_bytes(scratch_ctx)
    lib._lib.check(scratch_ctx.L.irsde_layernorm(scratch_ctx.h, 1 if bf else 0, _ptr(x), ctypes.byref(a), _ptr(y), B, N, C, info,
                                                 _stream()), scratch_ctx.h)
    torch.cuda.synchronize()
    worst = 0.0
    for b, p0, p1 in wins:
        ref, core, rel = ref_of(b, p0, p1)
        worst = max(worst, ((y[b * N + p0:b * N + p1, off:off + C].double() - ref).abs() / bound_of(ref, core, rel)).max().item())
    with capsys.disabled():
        _report(c, worst, wrong, "kind %d MAXV %d LPP %d PP %d" % tuple(info), _lib_bytes(scratch_ctx) - lb0)
    assert info[0] == c["expect"], tuple(info)
    assert out_before[0].shape[1] == 8 and out_before[1].shape[1] == 8
    assert torch.equal(_bits(y[:, :off]), _bits(out_before[0])) and torch.equal(_bits(y[:, off + C:]), _bits(out_before[1]))
    assert worst <= 1.0, worst


# ------------------------------------------------------------------------------------------------------------------
# GPU: attention
# ------------------------------------------------------------------------------------------------------------------
def _att_run(lib, ctx, c, qkv, out, cx):
    info = (ctypes.c_int32 * 4)()
    lb0 = _lib_bytes(ctx)
    kind = lib._lib.ATTN_FULL if c["full"] else lib._lib.ATTN_LINEAR
    lib._lib.check(ctx.L.irsde_attention(ctx.h, 1 if c["prec"] == "bf16" else 0, kind, _ptr(qkv), 384, 0, _ptr(out), 128, 0, None,
                                         0, _ptr(cx), c["B"], c["N"], info, _stream()), ctx.h)
    torch.cuda.synchronize()
    c["lib_bytes"] = _lib_bytes(ctx) - lb0
    return tuple(info)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ATT_CASES, ids=[c["id"] for c in ATT_CASES])
def test_attention_at_level_size_vs_fp64(lib, scratch_ctx, case, budget, capsys):
    c = case
    dev = _dev()
    B, N = c["B"], c["N"]
    bf = c["prec"] == "bf16"
    g = torch.Generator(device=dev).manual_seed(N + len(c["prec"]) + int(c["full"]))
    qkv = torch.randn(B * N, 384, generator=g, device=dev)
    # planted in the last chunk (64 pixels / keys): a dropped last chunk moves the result far past the bound
    if c["full"]:
        qkv[N - 1, 256:] = 2000.0
    else:
        mid = (-(-N // 64) * 17 // 37 + 5) * 64 + 9  # a pixel of a chunk that pass A's block 17 of 37 walks
        for n, vv in ((N - 1, 4.0), (mid, 3.0)):
            qkv[n, 128:256] = 12.0
            qkv[n, 256:] = vv
    if bf:
        qkv.copy_(qkv.bfloat16())
    out = torch.randn(B * N, 128, generator=g, device=dev)
    out.copy_(out.bfloat16())
    cx = torch.zeros(B, 4, 32, 32, device=dev)
    scale = 32 ** -0.5
    if c["full"]:
        rows = torch.cat([torch.arange(0, 64), torch.arange(N - 64, N), torch.arange(120, 136),
                          torch.from_numpy(np.random.default_rng(5).integers(0, N, 64))]).to(dev)
        q = qkv[rows, :128].double().view(-1, 4, 32).transpose(0, 1)        # [4, R, 32]
        k = qkv[:N, 128:256].double().view(N, 4, 32).transpose(0, 1)        # [4, N, 32]
        v = qkv[:N, 256:].double().view(N, 4, 32).transpose(0, 1)

        def ref_of(keys=N, sc=scale, head_shift=0):
            kk, vv = k[:, :keys].roll(head_shift, 0), v[:, :keys].roll(head_shift, 0)
            s = q @ kk.transpose(1, 2) * sc
            p = torch.exp(s - s.amax(-1, keepdim=True))
            S = p.sum(-1, keepdim=True)
            o = (p @ vv) / S
            return o, (p @ vv.abs()) / S, p, S

        o_ref, pv, p, S = ref_of()
        # |ds| <= 34 u sum|q k| scale; exp adds 4 u: each weight moves by <= (|ds| + ds_max + 4 u) relative
        ds = 34 * U * scale * (q.abs() @ k.abs().transpose(1, 2))
        dsm = ds.amax(-1, keepdim=True)
        sens = ((p * (ds + dsm + 4 * U)) @ v.abs()) / S + (dsm + 4 * U) * pv
        bound = _gamma(2 * N // 64 + 128) * pv * 4 + sens
        if bf:
            bound = bound + 2 ** -7 * (pv + o_ref.abs())  # P rounded to bf16 (sums of the rounded P), bf16 output
        wrong = [("dropped last chunk", ((ref_of(keys=N - 64)[0] - o_ref).abs() / bound).max().item()),
                 ("no 32^-0.5", ((ref_of(sc=1.0)[0] - o_ref).abs() / bound).max().item()),
                 ("other head", ((ref_of(head_shift=1)[0] - o_ref).abs() / bound).max().item())]
        info = _att_run(lib, scratch_ctx, c, qkv, out, cx)
        got = out[rows].double().view(-1, 4, 32).transpose(0, 1)
        worst = ((got - o_ref).abs() / bound).max().item()
        with capsys.disabled():
            _report(c, worst, wrong, "kernel %d" % info[0], c["lib_bytes"])
        assert info[0] == (4 if bf else 3), info
        assert worst <= 1.0, worst
        return
    # linear attention: the context over all N pixels in fp64, the hidden output on windows
    nblk = min(37, -(-N // 64))
    k = qkv[:N, 128:256].double()
    kmax = k.amax(0)
    pk = torch.exp(k - kmax)                                                   # [N, 128] = (head, d)
    Sk = pk.sum(0)
    v = qkv[:N, 256:].double()

    def ctx_of(keep=slice(None), inv=1.0 / N):
        """The context over the pixels `keep` selects (a boolean mask or a slice), times inv."""
        pp, vv = pk[keep], v[keep]
        pv = torch.einsum("nhd,nhe->hde", pp.reshape(-1, 4, 32), vv.reshape(-1, 4, 32))
        return pv / pp.sum(0).view(4, 32, 1) * inv

    def without(n0, n1):
        m = torch.ones(N, dtype=torch.bool, device=dev)
        m[n0:n1] = False
        return m

    ctx_ref = ctx_of()
    pabs = torch.einsum("nhd,nhe->hde", pk.view(N, 4, 32), v.abs().view(N, 4, 32)) / Sk.view(4, 32, 1) / N
    cb = (_gamma(2 * (-(-N // 64) // nblk + 1) * 64 + 2 * nblk + 64) * 4 + 64 * U) * pabs
    if bf:
        cb = cb + 2 ** -8 * pabs
    nch = -(-N // 64)
    b17 = (nch * 17 // 37 * 64, nch * 18 // 37 * 64)
    wrong = [("dropped last chunk", ((ctx_of(without(N - 64, N)) - ctx_ref).abs() / cb).max().item()),
             ("dropped a chunk of block 17", ((ctx_of(without(mid - 9, mid + 55)) - ctx_ref).abs() / cb).max().item()),
             ("dropped block 17's chunks", ((ctx_of(without(*b17)) - ctx_ref).abs() / cb).max().item()),
             ("1/N of the next level", ((ctx_of(inv=4.0 / N) - ctx_ref).abs() / cb).max().item())]
    info = _att_run(lib, scratch_ctx, c, qkv, out, cx)
    worst_ctx = ((cx[0].double() - ctx_ref).abs() / cb).max().item()
    worst = worst_ctx
    for p0 in (0, N - 64, N // 2 - 32, 777 * 64 + 5):
        q = qkv[p0:p0 + 64, :128].double().view(64, 4, 32)
        qs = torch.softmax(q, -1) * scale
        ref = torch.einsum("nhd,hde->nhe", qs, ctx_ref)
        bnd = torch.einsum("nhd,hde->nhe", qs, cb + 40 * U * ctx_ref.abs()) + 4 * U * ref.abs() + 1e-30
        if bf:
            bnd = bnd + 2 ** -8 * ref.abs() + 2 ** -10 * torch.einsum("nhd,hde->nhe", qs, ctx_ref.abs())
        got = out[p0:p0 + 64].double().view(64, 4, 32)
        worst = max(worst, ((got - ref).abs() / bnd).max().item())
    with capsys.disabled():
        _report(c, worst, wrong, "kernel %d nblk %d nchunks %d (context %.3f)" % (info[0], info[1], info[2], worst_ctx),
                c["lib_bytes"])
    assert info[0] == (2 if bf else 1) and info[1] == nblk and info[2] == -(-N // 64), info
    assert worst <= 1.0, worst


# ------------------------------------------------------------------------------------------------------------------
# GPU: the fused LinearAttention block over a whole level
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", BLOCK_CASES, ids=[c["id"] for c in BLOCK_CASES])
def test_linattn_block_at_level_size_vs_fp64(lib, scratch_ctx, case, capsys, budget):
    """The context is an online softmax over all N pixels scaled by 1/N, so it is checked through the block output with
    data that make it visible there: every pixel carries one channel pattern (plus noise) except two planted pixels with
    patterns of their own, the k rows of to_qkv give the planted pixels a key about 16 above the rest (each 15-40 % of the softmax weight),
    the v rows give the common pattern v = 0, so the context is the planted pixels' values, and they are scaled by N so that
    the context is O(0.1) against LayerNorm's eps.  xn must equal
    irsde_layernorm's bf16 output bit for bit; the reference takes it from there in fp64."""
    from test_gpu_linattn_fused import SCALE, TOL, _ln
    c = case
    dev = _dev()
    C, B, N = c["C"], c["B"], c["N"]
    ctx = scratch_ctx
    g = torch.Generator(device=dev).manual_seed(C + B + N % 9973)
    u = lambda *sh: torch.rand(*sh, generator=g, device=dev) * 2 - 1
    nch = -(-N // 64)
    mid = (nch * 17 // 37 + 5) * 64 + 9  # a pixel of a chunk that pass 1's block 17 of 37 walks
    a = torch.randn(C, generator=g, device=dev)
    plants = {mid: torch.randn(C, generator=g, device=dev), N - 1: torch.randn(C, generator=g, device=dev)}
    x = torch.randn(B * N, C, generator=g, device=dev).mul_(0.05).add_(a)
    for b in range(B):
        for n, pt in plants.items():
            x[b * N + n] = pt
    x.copy_(x.bfloat16())
    g1 = (0.5 + torch.rand(C, generator=g, device=dev)).contiguous()
    g2 = (0.5 + torch.rand(C, generator=g, device=dev)).contiguous()
    lnv = lambda v: _ln(v.double()[None], 1.0)[0][0] * g1.double()
    xa = lnv(a.bfloat16().float())
    X = torch.stack([xa] + [lnv(pt.bfloat16().float()) for pt in plants.values()])
    e = X.t() @ torch.linalg.solve(X @ X.t(), torch.tensor([0.0, 1.0, 1.0], device=dev, dtype=torch.float64))  # e.xn: 0, 1, 1
    wqkv = torch.empty(384, C, device=dev)
    wqkv[:128] = u(128, C) / math.sqrt(C) * 2
    wqkv[128:256] = (16.0 * (1 + 0.05 * u(128, 1))).double() * e[None] + 0.01 * u(128, C).double()
    wv = u(128, C).double()
    wqkv[256:] = (wv - (wv @ xa)[:, None] / (xa @ xa) * xa[None]) * (0.02 * N)
    wqkv = wqkv.contiguous()
    wout = (u(C, 128) / math.sqrt(128)).contiguous()
    W = wqkv.bfloat16().double()
    Wq, Wk, Wv = W[:128], W[128:256], W[256:]
    # xn = irsde_layernorm's bf16 output (kept as bf16: its values are bf16)
    y_ln = torch.zeros(B * N, C, device=dev)
    la = lib._lib.LnArgs(g=g1.data_ptr(), res=None, ss=None, in_pitch=C, in_off=0, res_pitch=0, res_off=0, out_pitch=C, out_off=0)
    lb0 = _lib_bytes(ctx)
    lib._lib.check(ctx.L.irsde_layernorm(ctx.h, 1, _ptr(x), ctypes.byref(la), _ptr(y_ln), B, N, C, None, _stream()), ctx.h)
    torch.cuda.synchronize()
    lib_peak = _lib_bytes(ctx) - lb0
    xn_ln = y_ln.bfloat16()
    assert torch.equal(xn_ln.float(), y_ln)
    del y_ln
    torch.cuda.empty_cache()

    # the fp64 context of each image: max, then sum of exp(k - max) v over all pixels, slab by slab
    def kv(b, n0, n1):
        xs = xn_ln[b * N + n0:b * N + n1].double()
        return xs @ Wk.t(), xs @ Wv.t()

    SL = 1 << 19
    kmax = torch.stack([torch.stack([(xn_ln[b * N + n0:b * N + min(N, n0 + SL)].double() @ Wk.t()).amax(0)
                                     for n0 in range(0, N, SL)]).amax(0) for b in range(B)])

    def sums(b, n0, n1):
        S = torch.zeros(128, device=dev, dtype=torch.float64)
        PV, PA = torch.zeros(4, 32, 32, device=dev, dtype=torch.float64), torch.zeros(4, 32, 32, device=dev, dtype=torch.float64)
        for s0 in range(n0, n1, SL):
            k, v = kv(b, s0, min(n1, s0 + SL))
            p = torch.exp(k - kmax[b])
            S += p.sum(0)
            PV += torch.einsum("nhd,nhe->hde", p.view(-1, 4, 32), v.view(-1, 4, 32))
            PA += torch.einsum("nhd,nhe->hde", p.view(-1, 4, 32), v.abs().view(-1, 4, 32))
        return S.view(4, 32, 1), PV, PA

    full = [sums(b, 0, N) for b in range(B)]
    ctx_ref = torch.stack([PV / S / N for S, PV, _ in full])
    ctx_abs = torch.stack([PA / S / N for S, _, PA in full])
    # pass 1 adds one 64-pixel MMA sum per chunk to each accumulator (and rescales it), then 37 records are merged
    gam = 4 * _gamma(2 * (nch // 37 + 1) + 64 + 2 * 37 + 16)
    wins = [(0, 0, 64), (B - 1, N - 64, N), (B - 1, N // 2 - 32, N // 2 + 32), (0, mid - 40, mid + 24)]
    x_w = {w: x[w[0] * N + w[1]:w[0] * N + w[2]].double() for w in wins}

    def out_ref(w, cx, ca, bo):
        b, p0, p1 = w
        q = (xn_ln[b * N + p0:b * N + p1].double() @ Wq.t()).view(-1, 4, 32)
        qs = q.softmax(-1) * SCALE
        hid = torch.einsum("nhd,hde->nhe", qs, cx[b]).reshape(-1, 128)
        hid_abs = torch.einsum("nhd,hde->nhe", qs, ca[b]).reshape(-1, 128)
        wo = wout.double()
        y = hid @ wo.t() + bo
        yh, rstd = _ln(y, 1.0)
        out = yh * g2.double() + x_w[w]
        dy = (TOL + gam) * (hid_abs @ wo.abs().t() + bo.abs())
        bound = (g2.double().abs() * rstd * (dy + dy.mean(1, keepdim=True) + yh.abs() * dy.pow(2).mean(1, keepdim=True).sqrt())
                 + 2 ** -8 * out.abs() + 1e-6)
        return out, bound, y

    y0 = out_ref(wins[0], ctx_ref, ctx_abs, torch.zeros(C, device=dev, dtype=torch.float64))[2]
    bout = (y0.std().item() * u(C)).contiguous()  # as large as y: 1/N of another level moves LayerNorm(y + b)
    bo = bout.double()

    def drop(b, n0, n1):
        """ctx with pixels n0 .. n1-1 of image b left out."""
        S, PV, PA = full[b]
        s, pv, _ = sums(b, n0, n1)
        cx = ctx_ref.clone()
        cx[b] = (PV - pv) / (S - s) / N
        return cx

    wb = wins[1]
    ref, bound, _ = out_ref(wb, ctx_ref, ctx_abs, bo)
    ratio = lambda cx: ((out_ref(wb, cx, ctx_abs, bo)[0] - ref).abs() / bound).max().item()
    b17 = (nch * 17 // 37 * 64, nch * 18 // 37 * 64)
    wrong = [("dropped last chunk", ratio(drop(B - 1, N - 64, N))),
             ("dropped a chunk of block 17", ratio(drop(B - 1, mid - 9, mid + 55))),
             ("dropped block 17's chunks", ratio(drop(B - 1, *b17))),
             ("1/N of the next level", ratio(ctx_ref * 4))]
    torch.cuda.empty_cache()
    out = torch.zeros(B * N, C, device=dev)
    xn = torch.full((B * N, C), float("nan"), device=dev)
    lb0 = _lib_bytes(ctx)
    lib._lib.check(ctx.L.irsde_linattn_block(ctx.h, _ptr(x), C, 0, _ptr(out), C, 0, _ptr(g1), _ptr(wqkv), _ptr(wout), _ptr(bout),
                                             _ptr(g2), _ptr(xn), B, N, C, _stream()), ctx.h)
    torch.cuda.synchronize()
    lib_peak = max(lib_peak, _lib_bytes(ctx) - lb0)
    for s0 in range(0, B * N, SL):
        assert torch.equal(_bits(xn[s0:s0 + SL]), _bits(xn_ln[s0:s0 + SL].float())), ("pass 1's xn differs from irsde_layernorm's", s0)
    got = {w: out[w[0] * N + w[1]:w[0] * N + w[2]].double() for w in wins}
    del out, xn, x
    worst = 0.0
    for w in wins:
        r, bd, _ = out_ref(w, ctx_ref, ctx_abs, bo)
        worst = max(worst, ((got[w] - r).abs() / bd).max().item())
    with capsys.disabled():
        _report(c, worst, wrong, "plant weight %.3f, context %.3g" % (
            (torch.exp(kv(B - 1, N - 1, N)[0] - kmax[B - 1]) / full[B - 1][0].view(128)).min().item(), ctx_ref.abs().max().item()),
            lib_peak)
    assert worst <= 1.0, worst


# ------------------------------------------------------------------------------------------------------------------
# GPU: NAFNet ops
# ------------------------------------------------------------------------------------------------------------------
def _naf_call(lib, ctx, c, kind, a, info=None):
    lb0 = _lib_bytes(ctx)
    lib._lib.check(ctx.L.irsde_nafnet_op(ctx.h, 1 if c["prec"] == "bf16" else 0, kind, ctypes.byref(a), c["B"], c["H"], c["W"],
                                         c["c"], info, _stream()), ctx.h)
    torch.cuda.synchronize()
    c["lib_bytes"] = _lib_bytes(ctx) - lb0


@pytest.mark.gpu
@pytest.mark.parametrize("case", NAF_CASES, ids=[c["id"] for c in NAF_CASES])
def test_nafnet_op_at_4096(lib, scratch_ctx, case, budget, capsys):
    c = case
    dev = _dev()
    B, H, W, cc = c["B"], c["H"], c["W"], c["c"]
    bf = c["prec"] == "bf16"
    g = torch.Generator(device=dev).manual_seed(H + cc + len(c["op"]) + int(bf))
    op = c["op"]
    ps = op == "PIXEL_SHUFFLE_ADD"
    Ho, Wo = (2 * H, 2 * W) if ps else (H, W)
    xw = 4 * cc if ps else cc if op == "ADD" else 2 * cc
    x = torch.randn(B, H, W, xw, generator=g, device=dev)
    if op == "DWGATE_SCA":
        # planted pooling chunks dominate the mean, so losing one shows: the last chunk, and chunk 65535 + 1000 (walked by
        # block y = 1000 on its second pass, chunk += gridDim.y)
        for ch in (H * W // 64 - 1, GRID_YZ + 1000):
            x[:, ch * 64 // W, ch * 64 % W:ch * 64 % W + 64] = 2000.0
    rnd = (lambda t: t.copy_(t.bfloat16())) if bf else (lambda t: t)
    rnd(x)
    y = rnd(torch.randn(B, Ho, Wo, cc, generator=g, device=dev)) if op in ("ADD", "PIXEL_SHUFFLE_ADD") else None
    opitch, ooff = cc + 8, 4
    out = rnd(torch.randn(B, Ho, Wo, opitch, generator=g, device=dev))
    sides = out[..., :ooff].clone(), out[..., ooff + cc:].clone()
    a = lib._lib.NafArgs()
    a.x, a.out = x.data_ptr(), out.data_ptr()
    a.x_pitch, a.x_off, a.out_pitch, a.out_off = xw, 0, opitch, ooff
    kinds = dict(DWGATE_SCA=0, SIMPLE_GATE=1, PIXEL_SHUFFLE_ADD=2, ADD=3)
    if y is not None:
        a.y, a.y_pitch, a.y_off = y.data_ptr(), cc, 0
    if op != "DWGATE_SCA":
        _naf_call(lib, scratch_ctx, c, kinds[op], a)
        got = out[..., ooff:ooff + cc]
        if op == "SIMPLE_GATE":
            ref = x[..., :cc] * x[..., cc:]
        elif op == "ADD":
            ref = x + y
        else:
            ref = x.view(B, H, W, cc, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(B, Ho, Wo, cc) + y
        if bf:
            ref = ref.bfloat16().float()
        with capsys.disabled():
            _report(c, 0.0, [], "bit-exact over %d elements" % got.numel(), c["lib_bytes"])
        assert torch.equal(_bits(got), _bits(ref)), (got - ref).abs().max().item()
        assert torch.equal(_bits(out[..., :ooff]), _bits(sides[0])) and torch.equal(_bits(out[..., ooff + cc:]), _bits(sides[1]))
        return
    w = torch.randn(2 * cc, 9, generator=g, device=dev) / 3
    bias = 0.1 * torch.randn(2 * cc, generator=g, device=dev)
    sw = torch.randn(cc, cc, generator=g, device=dev) / cc ** 0.5
    sb = 0.1 * torch.randn(cc, generator=g, device=dev)
    sca = torch.zeros(B, cc, device=dev)
    a.w, a.bias, a.sca_w, a.sca_b, a.sca = w.data_ptr(), bias.data_ptr(), sw.data_ptr(), sb.data_ptr(), sca.data_ptr()
    N = H * W
    nchunks = -(-N // 64)
    wk = w.double().view(2 * cc, 1, 3, 3)

    def gate_rows(b, r0, r1):
        """fp64 gate of rows r0..r1-1 of image b and its error bound (fp32 taps, the product, storage rounding)."""
        a0, a1 = max(0, r0 - 1), min(H, r1 + 1)
        xs = x[b, a0:a1].double().permute(2, 0, 1)[None]
        top, bot = (1 if r0 == 0 else 0), (1 if r1 == H else 0)
        xs = F.pad(xs, (1, 1, top, bot))
        acc = F.conv2d(xs, wk, bias.double(), groups=2 * cc)[0]
        aab = F.conv2d(xs.abs(), wk.abs(), bias.double().abs(), groups=2 * cc)[0]
        s = r0 - a0 - (1 - top)
        acc, aab = acc[:, s:s + r1 - r0], aab[:, s:s + r1 - r0]
        gte = acc[:cc] * acc[cc:]
        eg = _gamma(12) * (aab[:cc] * acc[cc:].abs() + acc[:cc].abs() * aab[cc:]) * 2 + 2 * U * gte.abs()
        if bf:
            eg = eg + 2 ** -8 * gte.abs()
        return gte.permute(1, 2, 0), eg.permute(1, 2, 0)

    # the SCA mean over all pixels in fp64, slab by slab, with per-row sums for the sums over chunk ranges
    sums = torch.zeros(B, cc, device=dev, dtype=torch.float64)
    sums_abs, errs = torch.zeros_like(sums), torch.zeros_like(sums)
    rowsum = torch.zeros(B, H, cc, device=dev, dtype=torch.float64)
    for b in range(B):
        for r0 in range(0, H, 256):
            gt, eg = gate_rows(b, r0, min(H, r0 + 256))
            rowsum[b, r0:r0 + gt.shape[0]] = gt.sum(1)
            sums_abs[b] += gt.abs().sum((0, 1))
            errs[b] += eg.sum((0, 1))
        sums[b] = rowsum[b].sum(0)

    def chunks_sum(b, c0, c1):
        """fp64 sum of the gate over pooling chunks c0 .. c1-1 of image b (64-pixel chunks, W % 64 == 0)."""
        p0, p1 = c0 * 64, c1 * 64
        if p0 // W == (p1 - 1) // W:
            r = p0 // W
            return gate_rows(b, r, r + 1)[0][0, p0 - r * W:p1 - r * W].sum(0)
        r0, r1 = -(-p0 // W), p1 // W
        tot = rowsum[b, r0:r1].sum(0) if r1 > r0 else torch.zeros(cc, device=dev, dtype=torch.float64)
        if p0 < r0 * W:
            tot = tot + gate_rows(b, r0 - 1, r0)[0][0, p0 - (r0 - 1) * W:].sum(0)
        if p1 > r1 * W:
            tot = tot + gate_rows(b, r1, r1 + 1)[0][0, :p1 - r1 * W].sum(0)
        return tot

    drop = lambda c0, c1: torch.stack([sums[b] - chunks_sum(b, c0, c1) for b in range(B)])

    def sca_of(s, n):
        return (s / n) @ sw.double().t() + sb.double()

    mean_err = (errs + _gamma(nchunks + 40) * sums_abs) / N + 2 * U * sums_abs / N
    sca_ref = sca_of(sums, N)
    sca_bound = mean_err @ sw.double().abs().t() + _gamma(cc + 8) * ((sums.abs() / N) @ sw.double().abs().t() + sb.double().abs())
    wrong = [("dropped last chunk", ((sca_of(drop(nchunks - 1, nchunks), N) - sca_ref).abs() / sca_bound).max().item()),
             ("dropped chunk 65535+1000", ((sca_of(drop(GRID_YZ + 1000, GRID_YZ + 1001), N) - sca_ref).abs() / sca_bound).max().item()),
             ("dropped second walk", ((sca_of(drop(GRID_YZ, 2 * GRID_YZ), N) - sca_ref).abs() / sca_bound).max().item()),
             ("1/N of the next level", ((sca_of(sums, N / 4) - sca_ref).abs() / sca_bound).max().item())]
    info = (ctypes.c_int32 * 4)()
    _naf_call(lib, scratch_ctx, c, 0, a, info)
    worst_sca = ((sca.double() - sca_ref).abs() / sca_bound).max().item()
    worst = worst_sca
    for b, r0, r1 in _windows(H, B, 1, 3, rows=2):
        gt, eg = gate_rows(b, r0, r1)
        ref = gt * sca_ref[b]
        bnd = gt.abs() * sca_bound[b] + eg * sca_ref[b].abs() + 2 * U * ref.abs() + (2 ** -8 * ref.abs() if bf else 0) + 1e-30
        got = out[b, r0:r1, :, ooff:ooff + cc].double()
        worst = max(worst, ((got - ref).abs() / bnd).max().item())
    with capsys.disabled():
        _report(c, worst, wrong, "chunk %d px, %d chunks (%d per block), %d SCA launches (sca %.3f)" % (
            info[0], info[1], -(-info[1] // GRID_YZ), info[2], worst_sca), c["lib_bytes"])
    assert tuple(info[:3]) == (64, nchunks, 2), tuple(info)
    assert torch.equal(_bits(out[..., :ooff]), _bits(sides[0])) and torch.equal(_bits(out[..., ooff + cc:]), _bits(sides[1]))
    assert worst <= 1.0, worst


# ------------------------------------------------------------------------------------------------------------------
# GPU: input packing and the in-kernel Philox past 2^31 bytes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", [PREP], ids=["prep_input fp32 16x(4090x4093 -> 4096^2) pitch 8, %s" % _gb(PREP["need"])])
def test_prep_input_past_2g_bytes(lib, case, budget, capsys):
    c = case
    dev = _dev()
    B, C, H, W, Hp, Wp, pitch = (c[k] for k in ("B", "C", "H", "W", "Hp", "Wp", "pitch"))
    g = torch.Generator(device=dev).manual_seed(11)
    xt = torch.randn(B, C, H, W, generator=g, device=dev)
    cond = torch.randn(B, C, H, W, generator=g, device=dev)
    out = torch.full((B, Hp, Wp, pitch), 3.0, device=dev)
    lib._lib.check(lib._lib.load().irsde_prep_input(0, _ptr(xt), _ptr(cond), _ptr(out), B, C, H, W, Hp, Wp, pitch, 1, 0, 0, 0, 0, 0,
                                                    _stream()))
    torch.cuda.synchronize()
    hmap = torch.tensor([h if h < H else 2 * (H - 1) - h for h in range(Hp)], device=dev)
    wmap = torch.tensor([w if w < W else 2 * (W - 1) - w for w in range(Wp)], device=dev)

    def ref_rows(b, r0, r1):
        xs = xt[b][:, hmap[r0:r1]][:, :, wmap].permute(1, 2, 0)
        cs = cond[b][:, hmap[r0:r1]][:, :, wmap].permute(1, 2, 0)
        return torch.cat([xs - cs, cs, torch.zeros(r1 - r0, Wp, pitch - 2 * C, device=dev)], -1)

    wins = _windows(Hp, B, H, 7)
    for b, r0, r1 in wins:
        assert torch.equal(_bits(out[b, r0:r1]), _bits(ref_rows(b, r0, r1))), (b, r0, r1)
    b, r0, r1 = wins[1]
    wrong = [("image B-2", float(not torch.equal(_bits(out[b, r0:r1]), _bits(ref_rows(b - 1, r0, r1))))),
             ("row - 1", float(not torch.equal(_bits(out[b, r0:r1]), _bits(ref_rows(b, r0 - 1, r1 - 1)))))]
    with capsys.disabled():
        _report(c | {"name": "prep_input %d elements" % out.numel()}, 0.0, [(k, 2.0 * v) for k, v in wrong], "bit-exact windows")


@pytest.mark.gpu
@pytest.mark.parametrize("case", [PHILOX], ids=["step_philox DSDE_SDE 43 x 3x4096^2 in place, %s" % _gb(PHILOX["need"])])
def test_step_philox_past_2g_elements(lib, case, budget, capsys):
    """DenoisingSDE's reverse_sde step (no mu) over 2.16e9 elements, x updated in place (out aliases x, as the sampler runs
    it), so that two buffers fit the budget; the windows' inputs are kept before the call."""
    c = case
    dev = _dev()
    B, E, t = c["B"], c["E"], 3
    mode = lib._lib.MODE_DSDE_SDE
    sde = lib.DenoisingSDE(25, 5, device=dev)
    g = torch.Generator(device=dev).manual_seed(13)
    x = torch.rand(B, E, device=dev, generator=g)
    noise = torch.randn(B, E, device=dev, generator=g)
    ctx = sde._ctx_for(x)
    lib._lib.check(ctx.L.irsde_set_image_base(ctx.h, 5), ctx.h)
    wins = [(0, 0, 4096), (B - 1, E - 4096, E), (B // 2, E // 2 - 2048, E // 2 + 2048)]
    x_before = {w: x[w[0], w[1]:w[2]].clone() for w in wins}
    lib._lib.check(ctx.L.irsde_step_philox(ctx.h, mode, _ptr(x), None, _ptr(noise), t, _ptr(x), B, E, SEED, _stream()), ctx.h)
    torch.cuda.synchronize()

    def step(b, j0, j1, z):
        o = torch.empty(j1 - j0, device=dev)
        xs, ns = x_before[(b, j0, j1)], noise[b, j0:j1].contiguous()
        lib._lib.check(ctx.L.irsde_step(ctx.h, mode, _ptr(xs), None, _ptr(ns), _ptr(z.float().contiguous()), t, _ptr(o), j1 - j0,
                                        _stream()), ctx.h)
        torch.cuda.synchronize()
        return o.double()

    def z_of(b, j0, j1, stream=t, **kw):
        return torch.from_numpy(philox_normals(SEED, [5 + b], E, stream, blocks=(j0 // 4, j1 // 4), **kw)[0]).to(dev)

    worst, wrong = 0.0, []
    for i, (b, j0, j1) in enumerate(wins):
        z = z_of(b, j0, j1)
        ref = step(b, j0, j1, z)
        k = (step(b, j0, j1, torch.ones_like(z)) - step(b, j0, j1, torch.zeros_like(z))).abs()
        bound = k * 2 ** -19 * (1 + z.abs()) + 2 ** -22 * ref.abs() + 1e-300
        if i == 1:
            for label, kw in _philox_mutations(t):
                wrong.append((label, ((step(b, j0, j1, z_of(b, j0, j1, **kw)) - ref).abs() / bound).max().item()))
        worst = max(worst, ((x[b, j0:j1].double() - ref).abs() / bound).max().item())
    lib._lib.check(ctx.L.irsde_set_image_base(ctx.h, 0), ctx.h)
    with capsys.disabled():
        _report(c | {"name": "step_philox DSDE_SDE %d elements per buffer" % x.numel()}, worst, wrong)
    assert worst <= 1.0, worst


# ------------------------------------------------------------------------------------------------------------------
# GPU: the imaging entries on 8 x 4096 x 4096 x 3
# ------------------------------------------------------------------------------------------------------------------
def _ssim_fp64(a, b, crop):
    """oracle.imaging_oracle.ssim on the GPU in fp64 (separable 11x11 Gaussian, valid region) for one HxWxC image pair."""
    from oracle.imaging_oracle import _gauss11
    k = torch.tensor(_gauss11(), dtype=torch.float64, device=a.device)
    x, y = (t[crop:t.shape[0] - crop, crop:t.shape[1] - crop].double().permute(2, 0, 1)[:, None] for t in (a, b))

    def filt(t):
        t = F.conv2d(t, k.view(1, 1, 11, 1))
        return F.conv2d(t, k.view(1, 1, 1, 11))

    C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2
    m1, m2 = filt(x), filt(y)
    s11, s22, s12 = filt(x * x) - m1 * m1, filt(y * y) - m2 * m2, filt(x * y) - m1 * m2
    return (((2 * m1 * m2 + C1) * (2 * s12 + C2)) / ((m1 * m1 + m2 * m2 + C1) * (s11 + s22 + C2))).mean().item()


@pytest.mark.gpu
@pytest.mark.parametrize("case", [IMG], ids=["imaging 8x4096x4096x3, %s" % _gb(IMG["need"])])
def test_imaging_entries_at_8x4096(lib, case, budget, capsys):
    from oracle import imaging_oracle as IO
    c = case
    dev = _dev()
    B, H, W, C = c["B"], c["H"], c["W"], c["C"]
    L = lib.imaging._bind()
    # the fp64 SSIM above is the oracle's SSIM
    g0 = np.random.default_rng(1)
    sa, sb = (g0.integers(0, 256, (48, 40, 3), dtype=np.uint8) for _ in range(2))
    small = _ssim_fp64(torch.from_numpy(sa).to(dev), torch.from_numpy(sb).to(dev), 2)
    assert abs(small - IO.ssim(sa[2:-2, 2:-2], sb[2:-2, 2:-2])) < 1e-12
    g = torch.Generator(device=dev).manual_seed(17)
    chw = torch.rand(B, C, H, W, generator=g, device=dev) * 1.2 - 0.1
    img = torch.empty(B, H, W, C, dtype=torch.uint8, device=dev)
    lib._lib.check(L.irsde_tensor2img_u8(_ptr(chw), _ptr(img), B, C, H, W, 0.0, 1.0, _stream()))
    back = torch.empty(B, C, H, W, device=dev)
    lib._lib.check(L.irsde_img2tensor_u8(_ptr(img), _ptr(back), B, C, H, W, _stream()))
    img2 = img.clone()
    img2[..., 0] = 255 - img2[..., 0]
    img2[:, ::7] //= 2
    crop = 4
    sums = torch.zeros(B, dtype=torch.int64, device=dev)
    lib._lib.check(L.irsde_sqerr_u8(_ptr(img), _ptr(img2), B, H, W, C, crop, _ptr(sums), _stream()))
    ws = torch.empty(L.irsde_ssim_workspace(B, H, W, C, crop), dtype=torch.float64, device=dev)
    ssim = torch.empty(B, dtype=torch.float64, device=dev)
    lib._lib.check(L.irsde_ssim_u8(_ptr(img), _ptr(img2), B, H, W, C, crop, _ptr(ws), _ptr(ssim), _stream()))
    torch.cuda.synchronize()
    for b in (0, B - 1):
        want = IO.tensor2img(chw[b].cpu().numpy())
        assert np.array_equal(img[b].cpu().numpy(), want), b
        assert torch.equal(_bits(back[b].cpu()), _bits(torch.from_numpy(IO.img2tensor(want)))), b
        d = img[b, crop:H - crop, crop:W - crop].long() - img2[b, crop:H - crop, crop:W - crop].long()
        assert int(sums[b]) == int((d * d).sum()), b
    wrong = []
    worst = 0.0
    for b in range(B):
        ref = _ssim_fp64(img[b], img2[b], crop)
        worst = max(worst, abs(ssim[b].item() - ref) / 1e-9)
        if b == B - 1:
            wrong += [("crop + 1", abs(_ssim_fp64(img[b], img2[b], crop + 1) - ref) / 1e-9),
                      ("image B-2", abs(_ssim_fp64(img[b - 1], img2[b - 1], crop) - ref) / 1e-9)]
    with capsys.disabled():
        _report(c | {"name": "imaging entries, %d-byte u8 buffers" % img.numel()}, worst, wrong,
                "tensor2img / img2tensor / sqerr bit-exact on images 0 and %d" % (B - 1))
    assert worst <= 1.0, worst


# ------------------------------------------------------------------------------------------------------------------
# GPU: shapes past a limit are refused at plan build and by the entries, before anything is allocated or launched
# ------------------------------------------------------------------------------------------------------------------
def _family(lib, name, dev):
    if name == "ConditionalUNet":
        net, levels = lib.ConditionalUNet(3, 3, 8, depth=2, precision="fp32"), 2
    elif name == "DenoisingUNet":
        net, levels = lib.DenoisingUNet(3, 3, 8, depth=2, precision="fp32"), 2
    elif name == "ConditionalNAFNet":
        net, levels = lib.ConditionalNAFNet(img_channel=3, width=8, middle_blk_num=1, enc_blk_nums=[1], dec_blk_nums=[1],
                                            precision="bf16"), 1
    else:
        net, levels = lib.UNet(3, 3, 8, ch_mult=[1, 2], embed_dim=4, precision="fp32"), 2
    return net.to(dev), levels


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["ConditionalUNet", "DenoisingUNet", "ConditionalNAFNet", "LatentUNet"])
def test_plan_build_refuses_shapes_past_the_limits(lib, family):
    dev = _dev()
    net, levels = _family(lib, family, dev)
    ctx = net.sync_weights(dev)
    s = 1 << levels
    b_max = 16383 if family == "DenoisingUNet" else 65535
    before = ctx.L.irsde_device_bytes(ctx.h)
    for B, H, W, what in ((b_max + 1, 16, 16, "65535"),               # gridDim.y / z
                          (1, 32768 + 1, 32768, "2^30"),              # H * W after padding
                          (1, 32768 - s + 1, 32768 + 1, "2^30")):     # padding alone passes the limit
        rc = ctx.L.irsde_plan_num_ops(ctx.h, B, H, W)
        assert rc == -1, (family, B, H, W, rc)
        msg = ctx.L.irsde_last_error(ctx.h).decode()
        assert what in msg, msg
        assert ctx.L.irsde_device_bytes(ctx.h) == before  # nothing was allocated
    assert ctx.L.irsde_plan_num_ops(ctx.h, 2, 16, 16) > 0  # the context still builds and runs plans
    x = torch.rand(2, 3, 16, 16, device=dev)
    if family in ("ConditionalUNet", "ConditionalNAFNet"):
        y = net(x, x, 3)
    elif family == "DenoisingUNet":
        y = net(x, 3)
    else:
        y = net(x)
    torch.cuda.synchronize()
    assert torch.isfinite(y).all()
    ctx.L.irsde_trim(ctx.h)


@pytest.mark.gpu
def test_entries_refuse_shapes_past_the_limits(lib, scratch_ctx):
    dev = _dev()
    ctx, L = scratch_ctx, lib.imaging._bind()
    # Only shapes whose launch would fail on its grid (y / z past 65535) if a check were missing: no call here can reach a
    # kernel that touches memory.  The H * W limit is refused at plan build above, where nothing is launched.  The buffers
    # still cover what the rest of a call could touch if its check were missing: the 1-D launches that would run (the
    # bf16 round trip of the block's 65536 x 64 output, the time MLP's 65536 rows, the SSIM reduction) stay inside them.
    buf = torch.zeros(1 << 22, device=dev)
    u8 = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
    calls = [
        ("full attention B", lambda: L.irsde_attention(ctx.h, 0, lib._lib.ATTN_FULL, _ptr(buf), 384, 0, _ptr(buf), 128, 0, None, 0,
                                                       None, 16384, 1, None, _stream()), "4 B"),
        ("linattn block B", lambda: L.irsde_linattn_block(ctx.h, _ptr(buf), 64, 0, _ptr(buf), 64, 0, _ptr(buf), _ptr(buf),
                                                          _ptr(buf), _ptr(buf), _ptr(buf), None, 65536, 1, 64, _stream()), "65535"),
        ("time embedding rows", lambda: L.irsde_time_embedding(0, _ptr(buf), 65536, 8, _ptr(buf), _ptr(buf), _ptr(buf), _ptr(buf),
                                                               _ptr(buf), _ptr(buf), 4, _ptr(buf), _ptr(buf), _stream()), "65535"),
        ("tensor2img B", lambda: L.irsde_tensor2img_u8(_ptr(buf), _ptr(u8), 65536, 3, 1, 1, 0.0, 1.0, _stream()), "65535"),
        ("img2tensor B", lambda: L.irsde_img2tensor_u8(_ptr(u8), _ptr(buf), 65536, 3, 1, 1, _stream()), "65535"),
        ("sqerr B", lambda: L.irsde_sqerr_u8(_ptr(u8), _ptr(u8), 65536, 1, 1, 1, 0, _ptr(buf), _stream()), "65535"),
        ("ssim B", lambda: L.irsde_ssim_u8(_ptr(u8), _ptr(u8), 65536, 16, 16, 1, 0, _ptr(buf), _ptr(buf), _stream()), "65535"),
    ]
    a = lib._lib.NafArgs()
    a.x, a.y, a.out = buf.data_ptr(), buf.data_ptr(), buf.data_ptr()
    a.w, a.bias, a.sca_w, a.sca_b, a.sca = (buf.data_ptr(),) * 5  # DWGATE_SCA: its grid has B in z
    a.x_pitch, a.y_pitch, a.out_pitch = 16, 16, 16
    calls += [("NAFNet op B", lambda: L.irsde_nafnet_op(ctx.h, 0, 0, ctypes.byref(a), 65536, 1, 1, 4, None, _stream()), "65535")]
    for label, call, what in calls:
        rc = call()
        assert rc == -1, (label, rc)
        msg = (L.irsde_last_error(None) or b"").decode()
        assert what in msg, (label, msg)
    torch.cuda.synchronize()
    assert torch.count_nonzero(buf) == 0 and torch.count_nonzero(u8) == 0
