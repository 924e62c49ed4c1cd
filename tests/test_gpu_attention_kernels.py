"""Every LayerNorm and attention kernel of attention.cu against an fp64 reference, through the standalone entries
irsde_layernorm and irsde_attention: the same launchers the launch plan calls, on views the plan gives them (channel slices
of wider NHWC buffers) and on the views that select the general kernels (odd pitches, unaligned offsets, widths that are not
a multiple of a 16-byte vector).

Each case names the kernels it must run and checks them through the `info` the call returns.  The reference follows the
reference module on the operands as the engine sees them (bf16-rounded for precision 1): LayerNorm with biased variance and
eps 1e-5 (module_util.py:70-79) with the NAFBlock time modulation and residual, LinearAttention (:163-178, including the
context, which the network never exposes, and its fold into the to_out weights) and Attention (:192-204).  Every bound
scales with an fp64 sum of the same terms in absolute value; before a kernel's output is compared, each of the case's wrong
references (a dropped pixel or key, a transposed context, another image's or head's operands, a wrong table row, ...) must
violate it.  Everything outside the written slice of every output buffer must come back bit-identical.

test_every_compiled_kernel_has_a_case runs without a GPU: it compiles attention.cu and fails when the object holds a kernel
that no case below names (or a case names one that no longer exists).
"""
import ctypes
import math
import os
import re
import shutil
import subprocess

import pytest
import torch

SCALE = 32 ** -0.5
LN_SCALAR, LN_VEC, LN_GEO = 0, 1, 2
K_LA_KV_F32, K_LA_KV_MMA, K_FULL, K_FULL_MMA = 1, 2, 3, 4  # info[0] of irsde_attention
LINEAR, LINEAR_FOLD, FULL = 0, 1, 2


# ------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------
def _ln(prec, expect, C, B, N, in_view=None, out_view=None, res_view=None, ss=None, t_row=1, note=""):
    """expect = (kind, MAXV, LPP, PP) from info; *_view = (pitch, channel offset) of the wide buffer (None: dense);
    ss = None | "shared" | "image"."""
    T = "float" if prec == "fp32" else "bf16"
    kind, mv, lpp, pp = expect
    kern = ("layernorm_scalar_kernel<%s>" % T if kind == LN_SCALAR else
            "layernorm_vec_kernel<%s,%d>" % (T, mv) if kind == LN_VEC else
            "layernorm_geo_kernel<%s,%d,%d,%d>" % (T, mv, lpp, pp))
    name = "%s %s C=%d B=%d N=%d%s" % (prec, kern, C, B, N, (" " + note) if note else "")
    return dict(name=name, prec=prec, expect=expect, kernels=[kern], C=C, B=B, N=N, in_view=in_view or (C, 0),
                out_view=out_view or (C, 0), res_view=res_view, ss=ss, t_row=t_row)


LN_CASES = [
    # ---- fp32
    _ln("fp32", (LN_SCALAR, 0, 0, 0), 30, 3, 41, in_view=(37, 5), out_view=(33, 1), res_view=(31, 1), ss="image", note="C % 4"),
    _ln("fp32", (LN_SCALAR, 0, 0, 0), 64, 3, 29, in_view=(70, 2), ss="shared", note="in_off 2"),
    _ln("fp32", (LN_VEC, 1, 4, 1), 16, 3, 45, in_view=(24, 8), out_view=(20, 4), res_view=(16, 0)),
    _ln("fp32", (LN_VEC, 2, 8, 1), 36, 3, 33, out_view=(40, 4), ss="image"),
    _ln("fp32", (LN_VEC, 4, 32, 1), 288, 3, 17, res_view=(296, 8)),
    _ln("fp32", (LN_VEC, 8, 32, 1), 640, 3, 13, in_view=(648, 8), ss="shared", t_row=3),
    _ln("fp32", (LN_VEC, 16, 32, 1), 2048, 3, 7, res_view=(2048, 0)),
    _ln("fp32", (LN_GEO, 1, 8, 2), 32, 3, 77, in_view=(48, 16), out_view=(64, 32), res_view=(40, 8)),
    _ln("fp32", (LN_GEO, 1, 16, 2), 64, 3, 55, ss="image", t_row=2),
    _ln("fp32", (LN_GEO, 1, 32, 2), 128, 3, 61, out_view=(256, 0), res_view=(256, 128)),
    _ln("fp32", (LN_GEO, 2, 32, 2), 256, 3, 45, ss="shared"),
    _ln("fp32", (LN_GEO, 4, 32, 1), 512, 3, 21, res_view=(512, 0), ss="image"),
    _ln("fp32", (LN_GEO, 8, 32, 1), 1024, 3, 19, in_view=(1088, 64), res_view=(1024, 0)),
    # ---- bf16
    _ln("bf16", (LN_SCALAR, 0, 0, 0), 20, 3, 41, in_view=(27, 3), out_view=(24, 2), res_view=(21, 1), ss="image", note="C % 8"),
    _ln("bf16", (LN_SCALAR, 0, 0, 0), 4352, 3, 9, res_view=(4352, 0), note="17 vectors per lane"),
    _ln("bf16", (LN_VEC, 1, 2, 1), 16, 3, 53, in_view=(32, 16), ss="shared"),
    _ln("bf16", (LN_VEC, 2, 8, 1), 72, 3, 35, res_view=(80, 8), ss="image"),
    _ln("bf16", (LN_VEC, 4, 32, 1), 576, 3, 15, out_view=(584, 8)),
    _ln("bf16", (LN_VEC, 8, 32, 1), 2048, 3, 9, ss="image", t_row=2),
    _ln("bf16", (LN_VEC, 16, 32, 1), 4096, 3, 5, res_view=(4096, 0)),
    _ln("bf16", (LN_GEO, 1, 8, 2), 64, 3, 77, in_view=(128, 64), out_view=(72, 8), ss="image"),
    _ln("bf16", (LN_GEO, 1, 16, 2), 128, 3, 55, res_view=(256, 128)),
    _ln("bf16", (LN_GEO, 1, 32, 2), 256, 3, 61, out_view=(512, 256), ss="shared"),
    _ln("bf16", (LN_GEO, 2, 32, 2), 512, 3, 45, res_view=(512, 0), ss="image"),
    _ln("bf16", (LN_GEO, 4, 32, 1), 1024, 3, 21, res_view=(1024, 0)),
]

LA_F32 = ["la_kv_kernel<float>", "la_combine8_kernel", "la_out_kernel<float>"]
LA_BF16 = ["la_kv_mma_kernel", "la_combine8_kernel", "la_out_kernel<bf16>"]
LA_FOLD = ["la_kv_mma_kernel", "la_combine8_kernel", "la_fold16_kernel"]


def _att(prec, kind, B, N, kernels, kern, qkv_view=(384, 0), out_view=(128, 0), Cout=0, note=""):
    """kern = info[0] the call must report; *_view = (pitch, channel offset) of the wide buffer."""
    name = "%s %s B=%d N=%d%s%s" % (prec, ["LINEAR", "LINEAR_FOLD", "FULL"][kind], B, N, " Cout=%d" % Cout if Cout else "",
                                     (" " + note) if note else "")
    return dict(name=name, prec=prec, kind=kind, B=B, N=N, kernels=kernels, kern=kern, qkv_view=qkv_view, out_view=out_view,
                Cout=Cout)


ATT_CASES = [
    # ---- linear attention, fp32
    _att("fp32", LINEAR, 3, 1, LA_F32, K_LA_KV_F32),
    _att("fp32", LINEAR, 3, 65, LA_F32, K_LA_KV_F32, qkv_view=(392, 4), note="pitched qkv"),
    _att("fp32", LINEAR, 3, 1900, LA_F32, K_LA_KV_F32, out_view=(136, 8), note="50x38, hidden into a slice"),
    _att("fp32", LINEAR, 2, 4096, LA_F32, K_LA_KV_F32),
    # ---- linear attention, bf16
    _att("bf16", LINEAR, 3, 64, LA_BF16, K_LA_KV_MMA),
    _att("bf16", LINEAR, 3, 2368, LA_BF16, K_LA_KV_MMA, qkv_view=(400, 8), note="37 chunks"),
    _att("bf16", LINEAR, 3, 2427, LA_BF16, K_LA_KV_MMA, out_view=(256, 128), note="38 chunks, last one partial"),
    _att("bf16", LINEAR, 2, 16384, LA_BF16, K_LA_KV_MMA),
    _att("bf16", LINEAR_FOLD, 2, 65536, LA_FOLD, K_LA_KV_MMA, Cout=128, note="27-28 chunks per block"),
    _att("bf16", LINEAR_FOLD, 3, 1024, LA_FOLD, K_LA_KV_MMA, Cout=72, note="partial fold block"),
    _att("bf16", LINEAR_FOLD, 3, 1024, LA_FOLD, K_LA_KV_MMA, Cout=512),
    # ---- full attention
    _att("fp32", FULL, 2, 1, ["fullattn_kernel<float>"], K_FULL),
    _att("fp32", FULL, 2, 65, ["fullattn_kernel<float>"], K_FULL, qkv_view=(389, 3), out_view=(131, 1), note="odd views"),
    _att("fp32", FULL, 2, 520, ["fullattn_kernel<float>"], K_FULL),
] + [_att("bf16", FULL, 1 if N >= 4096 else 2, N, ["fullattn_mma_kernel"], K_FULL_MMA,
          out_view=(256, 128) if N == 520 else (128, 0)) for N in (1, 63, 64, 65, 520, 1024, 4096)] + [
    _att("bf16", FULL, 2, 65, ["fullattn_kernel<bf16>"], K_FULL, qkv_view=(388, 2), note="qkv pitch 388"),
    _att("bf16", FULL, 2, 63, ["fullattn_kernel<bf16>"], K_FULL, out_view=(131, 1), note="odd hidden pitch"),
]


# ------------------------------------------------------------------------------------------------------------------
# (CPU) the cases name exactly the kernels the object holds
# ------------------------------------------------------------------------------------------------------------------
def _normalize(demangled):
    m = re.search(r"irsde::(\w+(?:<[^>]*>)?)", demangled)
    return m.group(1).replace("(int)", "").replace(" ", "").replace("__nv_bfloat16", "bf16")


def test_every_compiled_kernel_has_a_case(tmp_path):
    from test_conv_tc_sass import _build_module
    b = _build_module()
    nvcc = b.NVCC if os.path.isfile(b.NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    tools = os.path.dirname(nvcc)
    cuobjdump, cufilt = os.path.join(tools, "cuobjdump"), os.path.join(tools, "cu++filt")
    if not (os.path.isfile(cuobjdump) and os.path.isfile(cufilt)):
        pytest.skip("cuobjdump / cu++filt not available")
    obj = str(tmp_path / "attention.o")
    r = subprocess.run([nvcc] + b.FLAGS + ["-c", os.path.join(b.CSRC, "attention.cu"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    s = subprocess.run([cuobjdump, "-res-usage", obj], capture_output=True, text=True, check=True)
    mangled = re.findall(r"Function (\S+?):", s.stdout)
    dem = subprocess.run([cufilt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.split("\n")
    compiled = {_normalize(d) for d in dem if d.strip()}
    named = {k for c in LN_CASES + ATT_CASES for k in c["kernels"]}
    assert len(compiled) == 32, sorted(compiled)
    assert compiled == named, ("without a case", sorted(compiled - named), "not compiled", sorted(named - compiled))


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


def _same_outside(got, before, cols):
    """got / before: [rows, pitch] fp32; cols = (off, width) of the written slice: the rest must be bit-identical."""
    outside = torch.ones(got.shape[1], dtype=torch.bool, device=got.device)
    outside[cols[0]:cols[0] + cols[1]] = False
    return torch.equal(got[:, outside].view(torch.int32), before[:, outside].view(torch.int32))


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------------------------
def _ln_data(c, dev):
    g = _gen(c, dev)
    B, N, C = c["B"], c["N"], c["C"]
    P = B * N
    rnd = lambda *s: torch.randn(*s, generator=g, device=dev)
    uni = lambda *s: torch.rand(*s, generator=g, device=dev) * 2 - 1
    d = {}
    x = rnd(P, c["in_view"][0]) * (0.5 + torch.rand(P, 1, generator=g, device=dev)) + 0.5 * rnd(P, 1)
    # a near-constant pixel: variance comparable to eps, so eps = 1e-6 gives a visibly different answer
    io = c["in_view"][1]
    x[1, io:io + C] = 0.02 + 0.003 * rnd(C)
    d["x"] = _round(c, x)
    d["g"] = 0.5 + torch.rand(C, generator=g, device=dev)
    d["y"] = _round(c, rnd(P, c["out_view"][0]))
    d["res"] = _round(c, rnd(P, c["res_view"][0])) if c["res_view"] else None
    if c["ss"]:
        d["stride"] = 1 if c["ss"] == "image" else 0
        d["rows"] = c["t_row"] + (B - 1) * d["stride"] + 2      # room for the row after the last one used
        d["off_scale"], d["off_shift"] = 4, 4 + C + 3
        d["S"] = d["off_shift"] + C + 8                          # room for the table shifted by one channel
        d["ss"] = uni(d["rows"], d["S"])
    return d


def _ln_run(lib, ctx, c, d, N=None, **over):
    """One irsde_layernorm call; `over` replaces fields of the args struct (refusal test)."""
    a = lib._lib.LnArgs()
    a.g = d["g"].data_ptr()
    a.in_pitch, a.in_off = c["in_view"]
    a.out_pitch, a.out_off = c["out_view"]
    if c["res_view"]:
        a.res = d["res"].data_ptr()
        a.res_pitch, a.res_off = c["res_view"]
    if c["ss"]:
        a.ss, a.ss_rows, a.ss_S = d["ss"].data_ptr(), d["rows"], d["S"]
        a.off_scale, a.off_shift, a.ss_img_stride, a.t_row = d["off_scale"], d["off_shift"], d["stride"], c["t_row"]
    for k, v in over.items():
        setattr(a, k, v)
    y = d["y"].clone()
    info = (ctypes.c_int32 * 4)()
    rc = ctx.L.irsde_layernorm(ctx.h, _prec(c), _ptr(d["x"]), ctypes.byref(a), _ptr(y), c["B"], c["N"] if N is None else N,
                               c["C"], info, _stream())
    lib._lib.check(rc, ctx.h)
    torch.cuda.synchronize()
    return y, tuple(info)


def _ln_ref(c, d, eps=1e-5, unbiased=False, g_roll=False, res_next=False, rows=None, off_add=0, swap=False, mag=False):
    """fp64 reference [B*N, C]; the keyword arguments build the wrong references.  mag=True also returns the bound's
    magnitude |ln (scale + 1)| + |shift| + |res| and the cancellation scale rstd max|x| |g| |scale + 1| of each element."""
    B, N, C = c["B"], c["N"], c["C"]
    io = c["in_view"][1]
    x = d["x"][:, io:io + C].double()
    mean = x.mean(1, keepdim=True)
    var = x.var(1, unbiased=unbiased, keepdim=True)
    rstd = (var + eps).rsqrt()
    gg = d["g"].double()
    if g_roll:
        gg = torch.roll(gg, 1)
    ln = (x - mean) * rstd * gg
    y, m = ln, ln.abs()
    fac = torch.ones_like(ln)
    if c["ss"]:
        if rows is None:
            rows = [c["t_row"] + b * d["stride"] for b in range(B)]
        tab = d["ss"].double()[torch.tensor(rows, device=x.device).repeat_interleave(N)]
        os_, oh = d["off_scale"] + off_add, d["off_shift"] + off_add
        scale, shift = tab[:, os_:os_ + C], tab[:, oh:oh + C]
        if swap:
            scale, shift = shift, scale
        y = y * (scale + 1) + shift
        fac = (scale + 1).abs()
        m = ln.abs() * fac + shift.abs()
    if c["res_view"]:
        ro = c["res_view"][1]
        r = d["res"][:, ro:ro + C].double()
        if res_next:
            r = torch.roll(r, -1, dims=0)
        y = y + r
        m = m + r.abs()
    if not mag:
        return y
    cancel = rstd * x.abs().amax(1, keepdim=True) * gg.abs() * fac
    return y, m, cancel


def _ln_bound(c, m, cancel):
    """bf16: the output's rounding alone is up to 2^-8 |y|; fp32: 1e-5, plus the cancellation in x - mean."""
    tol = 2 ** -7 if c["prec"] == "bf16" else 1e-5
    return tol * m + 1e-5 * cancel


def _ln_mutations(c, d):
    m = [("eps 1e-6", dict(eps=1e-6)), ("gain shifted one channel", dict(g_roll=True))]
    if c["prec"] == "fp32" or c["C"] <= 32:  # where 1/(2C) exceeds the bound
        m.append(("unbiased variance", dict(unbiased=True)))
    if c["res_view"]:
        m.append(("residual from the next pixel", dict(res_next=True)))
    if c["ss"]:
        rows = [c["t_row"] + b * d["stride"] for b in range(c["B"])]
        m += [("row t+1", dict(rows=[r + 1 for r in rows])), ("row t-1", dict(rows=[r - 1 for r in rows])),
              ("scale and shift exchanged", dict(swap=True)), ("table shifted by one channel", dict(off_add=1))]
        if d["stride"]:
            m.append(("images 0 and 1 swap rows", dict(rows=[rows[1], rows[0]] + rows[2:])))
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("case", LN_CASES, ids=[c["name"] for c in LN_CASES])
def test_layernorm_vs_fp64(lib, scratch_ctx, case, capsys):
    c = case
    d = _ln_data(c, _dev())
    ref, m, cancel = _ln_ref(c, d, mag=True)
    bound = _ln_bound(c, m, cancel)
    # the bound must reject every wrong reference before it is used to accept the kernel
    for label, kw in _ln_mutations(c, d):
        r = _worst(_ln_ref(c, d, **kw) - ref, bound)
        assert r > 1.0, ("the bound does not see", label, r)
    y, info = _ln_run(lib, scratch_ctx, c, d)
    oo = c["out_view"][1]
    assert _same_outside(y, d["y"], (oo, c["C"])), "write outside the output slice"
    r = _worst(y[:, oo:oo + c["C"]].double() - ref, bound)
    with capsys.disabled():
        print("\n  info %-16s worst err / bound %.3f  %s" % (info, r, c["name"]), end="")
    assert info == c["expect"], (info, c["expect"])
    assert r <= 1.0, (c["name"], r)


# ------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------
def _la_partition(N):
    nchunks = (N + 63) // 64
    return max(1, min(37, nchunks)), nchunks


def _att_data(c, dev):
    """qkv [B*N, pitch] with the planted pixels / keys that make each wrong reference visible."""
    g = _gen(c, dev)
    B, N = c["B"], c["N"]
    qp, qo = c["qkv_view"]
    t = torch.randn(B, N, qp, generator=g, device=dev)
    v3 = t[..., qo:qo + 384].view(B, N, 3, 4, 32)  # [b, n, q|k|v, head, d]
    v3[:, :, 0] *= 1.5
    v3[:, :, 1] *= 1.5
    d = {}
    if c["kind"] == FULL:
        for j in {N - 1, 64} & set(range(N)):  # keys with a large norm: they dominate about half of the queries
            v3[:, j, 1] *= 4
    else:
        nblk, nchunks = _la_partition(N)
        d["p1"] = (nchunks // nblk) * 64 if nblk > 1 else None  # first pixel of block 1's chunk range
        # the last pixel and block 1's first pixel each own a k that is its channel's max by a clear margin
        k = v3[:, :, 1]
        for n, ds in ((N - 1, [3, 17]), (d["p1"], [9, 29])):
            if n is not None:
                lse = torch.logsumexp(k[:, :, :, ds], dim=1)
                k[:, n, :, ds] = lse + 3
        # the first pixels' q look at those channels, so the hidden output sees them too
        q = v3[:, :, 0]
        q[:, :8, :, [3, 17, 9, 29]] += 5
        k[:, :, 2, 5] = -80.0  # loses to no pixel: pixels past the image (-1e30) must still lose to it
    d["qkv"] = _round(c, t.reshape(B * N, qp))
    if c["kind"] == LINEAR_FOLD:
        d["wout"] = torch.randn(c["Cout"], 128, generator=g, device=dev) / 128 ** 0.5
        d["out"] = torch.randn(B * c["Cout"] * 128 + 1024, generator=g, device=dev)
    else:
        d["out"] = _round(c, torch.randn(B * N, c["out_view"][0], generator=g, device=dev))
    if c["kind"] != FULL:
        d["ctx"] = torch.randn(B * 4096 + 1024, generator=g, device=dev)
    return d


def _att_run(lib, ctx, c, d, B=None, N=None, prec=None, kind=None, qkv=None, qkv_view=None, out_view=None):
    """One irsde_attention call (keywords override the case: refusal and batch tests).  Returns out, ctx_out, info."""
    qp, qo = qkv_view or c["qkv_view"]
    op, oo = out_view or c["out_view"]
    out, cx = d["out"].clone(), d["ctx"].clone() if "ctx" in d else None
    info = (ctypes.c_int32 * 4)()
    rc = ctx.L.irsde_attention(ctx.h, _prec(c) if prec is None else prec, c["kind"] if kind is None else kind,
                               _ptr(d["qkv"] if qkv is None else qkv), qp, qo, _ptr(out), op, oo, _ptr(d.get("wout")),
                               c["Cout"], _ptr(cx), c["B"] if B is None else B, c["N"] if N is None else N, info, _stream())
    lib._lib.check(rc, ctx.h)
    torch.cuda.synchronize()
    return out, cx, tuple(info)


def _qkv(c, d):
    """q, k, v as [B, head, d, N] fp64."""
    B, N = c["B"], c["N"]
    qo = c["qkv_view"][1]
    t = d["qkv"][:, qo:qo + 384].double().view(B, N, 3, 4, 32).permute(2, 0, 3, 4, 1)
    return t[0], t[1], t[2]


def _la_ref(c, d, drop=None, transpose=False, next_image=False, k_over_channels=False):
    """fp64 LinearAttention: ctx [B,4,32,32], hidden [B*N,128] (or Mb [B,Cout,128] for the fold) and their |.| sums."""
    q, k, v = _qkv(c, d)
    B, N = c["B"], c["N"]
    if next_image:
        k, v = torch.roll(k, -1, 0), torch.roll(v, -1, 0)
    if drop is not None:
        keep = torch.tensor([n for n in range(N) if n != drop], device=k.device, dtype=torch.long)
        k, v = k[..., keep], v[..., keep]
    ks = k.softmax(dim=-2) if k_over_channels else k.softmax(dim=-1)
    ctx = torch.einsum("bhdn,bhen->bhde", ks, v) / N
    ctx_abs = torch.einsum("bhdn,bhen->bhde", ks, v.abs()) / N
    if transpose:
        ctx = ctx.transpose(-1, -2)
    if c["kind"] == LINEAR_FOLD:
        w = d["wout"].double().view(-1, 4, 32)  # [c, h, e]
        out = torch.einsum("che,bhde->bchd", w, ctx).reshape(B, -1, 128)
        out_abs = torch.einsum("che,bhde->bchd", w.abs(), ctx_abs).reshape(B, -1, 128)
    else:
        qs = q.softmax(dim=-2) * SCALE
        out = torch.einsum("bhde,bhdn->bnhe", ctx, qs).reshape(B * N, 128)
        out_abs = torch.einsum("bhde,bhdn->bnhe", ctx_abs, qs).reshape(B * N, 128)
    return ctx, ctx_abs, out, out_abs


def _fa_ref(c, d, drop=(), no_scale=False, other_head=False):
    """fp64 Attention: hidden [B*N,128] and sum_j attn |v|."""
    q, k, v = _qkv(c, d)
    B, N = c["B"], c["N"]
    if other_head:
        k = torch.roll(k, -1, 1)
    sim = torch.einsum("bhdi,bhdj->bhij", q * (1.0 if no_scale else SCALE), k)
    for j in drop:
        sim[..., j] = -math.inf
    attn = torch.nan_to_num(sim.softmax(dim=-1))  # every key dropped: no attention at all
    out = torch.einsum("bhij,bhdj->bihd", attn, v).reshape(B * N, 128)
    out_abs = torch.einsum("bhij,bhdj->bihd", attn, v.abs()).reshape(B * N, 128)
    return out, out_abs


def _att_mutations(c, d):
    B, N = c["B"], c["N"]
    if c["kind"] == FULL:
        m = [("key N-1 dropped", dict(drop=(N - 1,)))]
        if N > 64:
            m.append(("key 64 dropped", dict(drop=(64,))))
        if N > 1:  # one key: the output is its v whatever the scores
            m += [("32^-0.5 scale missing", dict(no_scale=True)), ("another head's keys", dict(other_head=True))]
        return m
    m = [("last pixel dropped", dict(drop=N - 1)), ("ctx transposed", dict(transpose=True)),
         ("k softmaxed over channels", dict(k_over_channels=True))]
    if d["p1"] is not None:
        m.append(("first pixel of block 1 dropped", dict(drop=d["p1"])))
    if B > 1:
        m.append(("image b reads image b+1's k and v", dict(next_image=True)))
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("case", ATT_CASES, ids=[c["name"] for c in ATT_CASES])
def test_attention_vs_fp64(lib, scratch_ctx, case, capsys):
    c = case
    d = _att_data(c, _dev())
    B, N = c["B"], c["N"]
    bf = c["prec"] == "bf16"
    tol_out = 2 ** -7 if bf else 2e-5
    tol_ctx = 2 ** -8 if bf else 2e-5
    if c["kind"] == FULL:
        ref, ref_abs = _fa_ref(c, d)
        for label, kw in _att_mutations(c, d):
            r = _worst(_fa_ref(c, d, **kw)[0] - ref, tol_out * ref_abs)
            assert r > 1.0, ("the bound does not see", label, r)
    else:
        ctx, ctx_abs, ref, ref_abs = _la_ref(c, d)
        for label, kw in _att_mutations(c, d):
            mctx, _, mout, _ = _la_ref(c, d, **kw)
            r_ctx = _worst(mctx - ctx, tol_ctx * ctx_abs)
            r_out = _worst(mout - ref, tol_out * ref_abs)
            assert r_ctx > 1.0 and r_out > 1.0, ("the bound does not see", label, r_ctx, r_out)
    out, cx, info = _att_run(lib, scratch_ctx, c, d)
    r_ctx = 0.0
    if c["kind"] == LINEAR_FOLD:
        n = B * c["Cout"] * 128
        assert torch.equal(out[n:].view(torch.int32), d["out"][n:].view(torch.int32)), "write past Mb"
        got = out[:n].view(B, c["Cout"], 128).double()
    else:
        op, oo = c["out_view"]
        assert _same_outside(out, d["out"], (oo, 128)), "write outside the hidden slice"
        got = out[:, oo:oo + 128].double()
    r = _worst(got - ref, tol_out * ref_abs)
    if c["kind"] != FULL:
        assert torch.equal(cx[B * 4096:].view(torch.int32), d["ctx"][B * 4096:].view(torch.int32)), "write past ctx"
        r_ctx = _worst(cx[:B * 4096].view(B, 4, 32, 32).double() - ctx, tol_ctx * ctx_abs)
    with capsys.disabled():
        print("\n  info %-18s worst err / bound: out %.3f ctx %.3f  %s" % (info, r, r_ctx, c["name"]), end="")
    if c["kind"] == FULL:
        assert info == (c["kern"], 0, 0, 0), info
    else:
        assert info == (c["kern"],) + _la_partition(N) + (0,), info
    assert r <= 1.0 and r_ctx <= 1.0, (c["name"], r, r_ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,N", [("fp32", 1900), ("bf16", 2427)])
def test_linear_attention_image_independent_of_batch(lib, scratch_ctx, prec, N):
    """ctx and hidden of image 1 in a batch of 3 equal those of the same image run alone, bit for bit: the k,v pass's
    chunk partition (and with it the summation order) does not depend on the batch."""
    c = _att(prec, LINEAR, 3, N, [], 0)
    d = _att_data(c, _dev())
    out, cx, _ = _att_run(lib, scratch_ctx, c, d)
    one = dict(qkv=d["qkv"][N:2 * N].clone(), out=d["out"][N:2 * N].clone(), ctx=d["ctx"][:4096 + 1024].clone())
    out1, cx1, _ = _att_run(lib, scratch_ctx, c, one, B=1)
    assert torch.equal(cx[4096:2 * 4096].view(torch.int32), cx1[:4096].view(torch.int32))
    assert torch.equal(out[N:2 * N].view(torch.int32), out1.view(torch.int32))


@pytest.mark.gpu
def test_entries_refuse_bad_arguments(lib, scratch_ctx):
    """Host-side validation: each call below describes a view outside its pitch, a time row past the table, a linear-
    attention view the 16-byte kernels cannot load, the fold in fp32 or an empty image, and must be refused.  Every buffer
    has a generous tail, so a check that let an out-of-pitch call through would still stay inside the allocations; the
    misaligned views are refused again by the launchers themselves."""
    dev = _dev()
    tail = lambda t: torch.cat([t.reshape(-1), torch.zeros(1 << 18, device=dev)])
    c = LN_CASES[0]  # fp32 scalar, pitched views, per-image rows
    d = _ln_data(c, dev)
    d.update(x=tail(d["x"]), y=tail(d["y"]), res=tail(d["res"]), ss=tail(d["ss"]))
    C, B = c["C"], c["B"]
    bad = [dict(in_off=c["in_view"][0] - C + 1),              # input past its pitch
           dict(out_off=-1),                                  # negative offset
           dict(res_pitch=C - 1, res_off=0),                  # residual wider than its pitch
           dict(t_row=d["rows"] - (B - 1)),                   # the last image's row is past the table
           dict(off_shift=d["S"] - C + 1)]                    # shift columns past the row
    for kw in bad:
        with pytest.raises(lib._lib.IrsdeError):
            _ln_run(lib, scratch_ctx, c, d, **kw)
    with pytest.raises(lib._lib.IrsdeError):
        _ln_run(lib, scratch_ctx, c, d, N=0)
    _ln_run(lib, scratch_ctx, c, d)  # the unmodified call is accepted

    c = _att("fp32", LINEAR, 2, 65, [], 0, qkv_view=(392, 4), out_view=(136, 8), Cout=64)
    d = _att_data(c, dev)
    d.update(qkv=tail(d["qkv"]), out=tail(d["out"]), ctx=tail(d["ctx"]))
    d["wout"] = torch.randn(64, 128, device=dev)
    bad = [dict(qkv_view=(392, 12)),                          # q|k|v past the pitch
           dict(out_view=(136, 12)),                          # hidden past the pitch
           dict(kind=FULL, out_view=(130, 3)),                # hidden past the pitch, full attention
           dict(qkv_view=(392, 2)),                           # fp32 view not on 16 bytes
           dict(qkv_view=(390, 4)),                           # fp32 pitch not a multiple of 16 bytes
           dict(out_view=(136, 6)),                           # fp32 hidden view not on 16 bytes
           dict(prec=1, qkv_view=(388, 0)),                   # bf16 pitch not a multiple of 16 bytes
           dict(prec=1, qkv_view=(392, 4)),                   # bf16 view not on 16 bytes
           dict(prec=1, kind=LINEAR_FOLD, qkv_view=(388, 0)),
           dict(kind=LINEAR_FOLD),                            # the fold is the bf16 path
           dict(N=0), dict(kind=FULL, N=0)]
    for kw in bad:
        with pytest.raises(lib._lib.IrsdeError):
            _att_run(lib, scratch_ctx, c, d, **kw)
    _att_run(lib, scratch_ctx, c, d)  # the unmodified call is accepted
