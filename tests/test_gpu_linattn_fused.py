"""The fused Residual(PreNorm(LinearAttention)) block of the bf16 path (linattn_fused.cu: LayerNorm + k,v projection + the
context partials; combine; fold; LayerNorm + q projection + q softmax + to_out + LayerNorm + residual) against an fp64
restatement of module_util.py:150-178, through the standalone entry irsde_linattn_block, which runs the launchers the plan
builder calls.

The reference takes the operands as the engine sees them: x and the to_qkv weight rounded to bf16, and xn = LayerNorm(x)
rounded to bf16 (the first pass's xn tile must equal irsde_layernorm's bf16 output bit for bit, checked here).  From there it
is fp64.  The bound on the block output scales with fp64 sums of the same terms in absolute value, carried through the
second LayerNorm (an error d in y moves the output by about |g2| rstd (|d| + mean|d| + |y_hat| rms(d))), plus the bf16
rounding of the output.  Before the kernels' output is compared, each wrong reference (a wrong gain, another image's
folded context, the residual dropped) must violate it.  Everything outside the written slice of the output buffer must come
back bit-identical.
"""
import ctypes
import math

import pytest
import torch

SCALE = 32 ** -0.5
TOL = 2 ** -6

# (C, B, N, (x pitch, x channel offset), (out pitch, out channel offset), note)
CASES = [
    (64, 2, 256 * 256, (64, 0), (128, 64), "256x256: every pass-1 block streams 27-28 full chunks; out = the upper half of a concat"),
    (128, 2, 256 * 256, (128, 0), (256, 128), "256x256, out = the upper half of a concat"),
    (64, 3, 777, (72, 8), (66, 2), "N % 64 != 0 and N % 16 != 0, pitched views"),
    (128, 3, 1000, (136, 8), (384, 128), "N % 64 != 0, pitched views"),
    (128, 2, 4096, (256, 128), (130, 2), "x at a channel offset"),
]


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


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bf(t):
    return t.bfloat16().float()


def _data(C, B, N, xv, ov, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    u = lambda *s: torch.rand(*s, generator=g, device=dev) * 2 - 1
    d = dict(
        # a channel pattern of its own per image: the images' contexts differ, so another image's context is visible
        x=_bf((torch.randn(B, N, xv[0], generator=g, device=dev) + 4 * torch.randn(B, 1, xv[0], generator=g, device=dev))
              .reshape(B * N, xv[0])),
        out=_bf(torch.randn(B * N, ov[0], generator=g, device=dev)),
        g1=0.5 + torch.rand(C, generator=g, device=dev),
        g2=0.5 + torch.rand(C, generator=g, device=dev),
        wqkv=u(384, C) / math.sqrt(C) * 2,
        wout=u(C, 128) / math.sqrt(128),
        bout=u(C) * 0.03 / N,  # the context carries 1/N (module_util.py:172): a larger bias would hide it in LayerNorm(y)
    )
    return {k: v.contiguous() for k, v in d.items()}


def _ln(x, g):
    mu = x.mean(1, keepdim=True)
    var = ((x - mu) ** 2).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    return (x - mu) * rstd * g, rstd


def _ref(d, C, B, N, xv, xn, gain=None, next_image=False, residual=True):
    """fp64 block output [B*N, C] and its bound."""
    x = d["x"][:, xv[1]:xv[1] + C].double()
    w = _bf(d["wqkv"]).double()
    qkv = xn.double() @ w.t()
    q, k, v = qkv.view(B, N, 3, 4, 32).permute(2, 0, 3, 4, 1)
    ks = k.softmax(dim=-1)
    ctx = torch.einsum("bhdn,bhen->bhde", ks, v) / N
    ctx_abs = torch.einsum("bhdn,bhen->bhde", ks, v.abs()) / N
    if next_image:
        ctx = torch.roll(ctx, -1, 0)
    qs = q.softmax(dim=-2) * SCALE
    hid = torch.einsum("bhde,bhdn->bnhe", ctx, qs).reshape(B * N, 128)
    hid_abs = torch.einsum("bhde,bhdn->bnhe", ctx_abs, qs).reshape(B * N, 128)
    wo, bo = d["wout"].double(), d["bout"].double()
    y = hid @ wo.t() + bo
    y_abs = hid_abs @ wo.abs().t() + bo.abs()
    g2 = (d["g2"] if gain is None else gain).double()
    yh, rstd = _ln(y, 1.0)
    out = yh * g2 + (x if residual else 0.0)
    dy = TOL * y_abs
    bound = (g2.abs() * rstd * (dy + dy.mean(1, keepdim=True) + yh.abs() * dy.pow(2).mean(1, keepdim=True).sqrt())
             + 2 ** -8 * out.abs() + 1e-6)
    return out, bound


def _run(lib, ctx, d, C, B, N, xv, ov, want_xn):
    out = d["out"].clone()
    xn = torch.full((B * N, C), float("nan"), device=out.device) if want_xn else None
    L = ctx.L
    lib._lib.check(L.irsde_linattn_block(ctx.h, _ptr(d["x"]), xv[0], xv[1], _ptr(out), ov[0], ov[1], _ptr(d["g1"]),
                                         _ptr(d["wqkv"]), _ptr(d["wout"]), _ptr(d["bout"]), _ptr(d["g2"]), _ptr(xn), B, N, C,
                                         _stream()), ctx.h)
    torch.cuda.synchronize()
    return out, xn


def _layernorm_bf16(lib, ctx, d, C, B, N, xv):
    y = torch.zeros(B * N, C, device=d["x"].device)
    a = lib._lib.LnArgs(g=d["g1"].data_ptr(), res=None, ss=None, in_pitch=xv[0], in_off=xv[1], res_pitch=0, res_off=0,
                        out_pitch=C, out_off=0)
    info = (ctypes.c_int32 * 4)()
    lib._lib.check(ctx.L.irsde_layernorm(ctx.h, 1, _ptr(d["x"]), ctypes.byref(a), _ptr(y), B, N, C, info, _stream()), ctx.h)
    torch.cuda.synchronize()
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=["C=%d B=%d N=%d %s" % (c[0], c[1], c[2], c[5]) for c in CASES])
def test_linattn_block_vs_fp64(lib, scratch_ctx, case, capsys):
    C, B, N, xv, ov, note = case
    dev = _dev()
    d = _data(C, B, N, xv, ov, dev, seed=C * 7919 + B * 31 + N)
    xn_ln = _layernorm_bf16(lib, scratch_ctx, d, C, B, N, xv)
    ref, bound = _ref(d, C, B, N, xv, xn_ln)
    mutations = [("wrong gain (g1 for g2)", dict(gain=d["g1"])), ("residual dropped", dict(residual=False))]
    if B > 1:
        mutations.append(("image b uses image b+1's folded context", dict(next_image=True)))
    seen = [(label, ((_ref(d, C, B, N, xv, xn_ln, **kw)[0] - ref).abs() / bound).max().item()) for label, kw in mutations]
    out, xn = _run(lib, scratch_ctx, d, C, B, N, xv, ov, want_xn=True)
    r = ((out[:, ov[1]:ov[1] + C].double() - ref).abs() / bound).max().item()
    with capsys.disabled():
        print("\n  worst err / bound %.3f, wrong references %s  C=%d B=%d N=%d" % (r, ["%.1f" % m for _, m in seen], C, B, N), end="")
    for label, m in seen:  # the bound must reject every wrong reference before it is used to accept the kernels
        assert m > 1.0, ("the bound does not see", label, m)
    assert torch.equal(xn.view(torch.int32), xn_ln.view(torch.int32)), "pass 1's xn differs from irsde_layernorm's bf16 output"
    outside = torch.ones(ov[0], dtype=torch.bool, device=dev)
    outside[ov[1]:ov[1] + C] = False
    assert torch.equal(out[:, outside].view(torch.int32), d["out"][:, outside].view(torch.int32)), "write outside the slice"
    assert r <= 1.0, r


@pytest.mark.gpu
def test_linattn_block_refuses_bad_arguments(lib, scratch_ctx):
    dev = _dev()
    C, B, N = 64, 1, 64
    d = _data(C, B, N, (64, 0), (64, 0), dev, seed=1)
    L, h = scratch_ctx.L, scratch_ctx.h

    def call(C=C, xv=(64, 0), ov=(64, 0)):
        return L.irsde_linattn_block(h, _ptr(d["x"]), xv[0], xv[1], _ptr(d["out"]), ov[0], ov[1], _ptr(d["g1"]), _ptr(d["wqkv"]),
                                     _ptr(d["wout"]), _ptr(d["bout"]), _ptr(d["g2"]), None, B, N, C, _stream())
    before = d["out"].clone()
    assert call(C=256) != 0          # the unfused path's width
    assert call(xv=(64, 8)) != 0     # view past its pitch
    assert call(xv=(68, 4)) != 0     # input offset not on 16 bytes of bf16
    assert call(ov=(65, 1)) != 0     # odd output offset
    torch.cuda.synchronize()
    assert torch.equal(d["out"], before)
