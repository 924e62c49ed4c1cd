"""Every entry point with a `stream` argument works in its caller's stream order on a non-blocking stream.

The rest of the suite runs on the legacy default stream, which orders itself against every blocking stream, so it cannot see
a call that does part of its work on the legacy stream, reads an input before earlier work on the caller's stream wrote it,
or shares context buffers with a call on another stream.  Here the caller's stream is created non-blocking, and a sleep
kernel stalls one stream for 20-150 ms.  The stall fixes the order in which the streams run, so each scenario is
deterministic: nothing loops and nothing races.

Every result is compared bit for bit with the same call on the legacy stream (same kernels, same inputs; the fp64 suites
pin the numerics), after that reference has given equal bits twice.  Input buffers hold a different valid input until the
producer on the stream overwrites them, so a read that comes too early gives a plausible wrong answer rather than NaN.

  S1  producer on s: stall s, write the inputs on s, call on s, copy the outputs on s;
  S2  legacy stalled, everything warm: the call on s must not wait for the legacy stream, and the hot-path entries must
      return while work on s is still pending (they never synchronize);
  S3  cold calls with the legacy stream stalled: a new (B, H, W), a first graph capture, a chain that grows the time table;
  S4  weights produced on a stream and uploaded from device memory;
  S5  two streams on one context;
  S6  the Python front-ends under torch.cuda.stream(s).
The CPU tests check that every stream entry has an S1/S2 case and that every legacy-stream call in csrc/ is accounted for."""
import ctypes
import glob
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "image-restoration-sde_b200")
HEADER = os.path.join(ROOT, "include", "irsde_b200.h")

# ---- case registry (read by the CPU coverage test) -------------------------------------------------------------------
CASES = {}   # name -> (builder(env) -> (good inputs, alt inputs, outs(bufs), call(bufs, outs, stream)), symbols, hot)


def case(name, symbols, hot=True):
    """hot: the entry neither synchronizes nor frees memory, so the host call returns while its stream still has work."""
    def deco(fn):
        CASES[name] = (fn, tuple(symbols), hot)
        return fn
    return deco


# stream entries without an S1/S2 case here
EXCLUDED = {
    "irsde_broadcast_weights": "NCCL collective: needs a communicator over two or more GPUs (tests/test_gpu_multi.py)",
    "irsde_gather": "NCCL collective: needs a communicator over two or more GPUs (tests/test_gpu_multi.py)",
}


# ---- CPU: coverage ---------------------------------------------------------------------------------------------------
def _stream_entries():
    import importlib.util
    spec = importlib.util.spec_from_file_location("irsde_lib_syms", os.path.join(PKG, "_lib.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)   # _lib imports ctypes and os only: no library, no GPU
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    out = []
    for sym in mod.SYMBOLS:
        m = re.search(r"\b%s\s*\(([^;]*)\)\s*;" % sym, text)
        assert m, "%s is not declared in the header" % sym
        if m.group(1).replace("\n", " ").strip().endswith("void* stream"):
            out.append(sym)
    return out


def test_every_stream_entry_has_a_case():
    entries = _stream_entries()
    assert len(entries) >= 20, entries
    covered = {s for _, syms, _ in CASES.values() for s in syms}
    missing = [s for s in entries if s not in covered and s not in EXCLUDED]
    assert not missing, "stream entries without an S1/S2 case: %s" % missing
    assert not (set(EXCLUDED) & covered)
    assert set(EXCLUDED) <= set(entries)
    assert covered <= set(entries), covered - set(entries)


# Every call in csrc/*.cu that runs on the legacy stream, with the reason it is safe: (file, function, call) -> reason.
LEGACY_CALLS = {
    ("engine.cu", "upload_coeffs", "cudaMemcpy"):
        "irsde_set_schedule / irsde_set_coeffs: between two cudaDeviceSynchronize calls",
    ("engine.cu", "build", "cudaMemset"):
        "the bf16 stem's zero border of a new plan: build_plan synchronizes the device before the plan is used",
    ("engine.cu", "build_plan", "cudaMemset"):
        "d_zero of a new plan: followed by cudaDeviceSynchronize before the plan is used",
    ("engine.cu", "irsde_load_tensor", "cudaMemcpy"):
        "between two cudaDeviceSynchronize calls",
    ("engine.cu", "irsde_finalize_weights", "cudaMemcpy"):
        "time-modulation matrices: followed by cudaDeviceSynchronize",
    ("engine.cu", "irsde_finalize_weights", "pack_weight"):
        "weight repacking: followed by cudaDeviceSynchronize",
    ("conv_tc.cu", "tc_conv_launch", "cudaMemcpy"):
        "IRSDE_TC_DEBUG counter dump after cudaStreamSynchronize (debug aid)",
}


def _top_args(s):
    """Top-level comma-separated arguments of s (parentheses and brackets nest)."""
    out, depth, cur = [], 0, ""
    for ch in s:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            out.append(cur.strip())
            cur = ""
        else:
            cur += ch
    out.append(cur.strip())
    return out


def _call_body(text, open_paren):
    depth = 0
    for i in range(open_paren, len(text)):
        if text[i] == "(":
            depth += 1
        elif text[i] == ")":
            depth -= 1
            if depth == 0:
                return text[open_paren + 1:i]
    raise AssertionError("unbalanced call")


_FUNC = re.compile(r"^ {0,2}(?!if\b|for\b|while\b|switch\b|return\b|else\b)[A-Za-z_][\w:<>\*&, ]*?\b(\w+)\s*\([^;]*$")


def _function_at(lines, lineno):
    for i in range(lineno, -1, -1):
        ln = lines[i]
        if ln.startswith(("#", "//", "}", " //", "  //")) or ln.strip().startswith("//"):
            continue
        m = _FUNC.match(ln)
        if m and "=" not in ln.split("(")[0]:
            return m.group(1)
    return "?"


def _legacy_calls():
    found = set()
    for path in sorted(glob.glob(os.path.join(PKG, "csrc", "*.cu"))):
        fname = os.path.basename(path)
        text = open(path).read()
        lines = text.split("\n")
        line_of = lambda pos: text.count("\n", 0, pos)

        def add(pos, what):
            ln = lines[line_of(pos)]
            if "//" in ln and ln.index("//") < pos - text.rfind("\n", 0, pos) - 1:
                return   # inside a comment
            found.add((fname, _function_at(lines, line_of(pos)), what))

        for m in re.finditer(r"\b(cudaMemcpy|cudaMemset)\(", text):
            add(m.start(), m.group(1))
        for m in re.finditer(r"<<<(.*?)>>>", text, flags=re.S):
            a = _top_args(m.group(1))
            if len(a) < 4 or a[3] in ("0", "nullptr", "NULL", "(cudaStream_t)0"):
                add(m.start(), "<<<>>>")
        for m in re.finditer(r"\bpack_weight(?:<\w+>)?\(", text):
            a = _top_args(_call_body(text, m.end() - 1))
            if len(a) == 9 and a[8] in ("0", "nullptr", "NULL"):
                add(m.start(), "pack_weight")
        for m in re.finditer(r"\bpdl_launch\(", text):
            body = _call_body(text, m.end() - 1)
            kern = re.match(r"\s*[\w:]+(?:<[^()]*?>)?\s*,", body)   # the kernel, template arguments included
            if not kern:
                continue   # the definition in common.cuh
            a = _top_args(body[kern.end():])   # grid, block, smem, stream, kernel arguments...
            if len(a) >= 4 and a[3] in ("0", "nullptr", "NULL"):
                add(m.start(), "pdl_launch")
    return found


def test_no_unaccounted_legacy_stream_calls():
    found = _legacy_calls()
    extra = sorted(found - set(LEGACY_CALLS))
    assert not extra, "legacy-stream calls without a reason in LEGACY_CALLS: %s" % extra
    stale = sorted(set(LEGACY_CALLS) - found)
    assert not stale, "LEGACY_CALLS entries that no longer match any call: %s" % stale


def test_legacy_scan_finds_what_it_should():
    """The scanner itself: each pattern it looks for is found, and a launch on the caller's stream is not."""
    src = ("int f(cudaStream_t st) {\n  k<<<1, 32>>>(x);\n  k<<<1, 32, 0, st>>>(x);\n  // cudaMemset(p, 0, 4);\n"
           "  pack_weight<bf16>(l, w, o, 1, 2, 3, 3, 1, 0);\n  pdl_launch(kern<T, 2>, g, 256, 0, 0, x);\n"
           "  pdl_launch(kern<T, 2>, g, 256, 0, st, x);\n  cudaMemcpy(a, b, 4, cudaMemcpyDefault);\n}\n")
    import tempfile
    global PKG
    saved = PKG
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "csrc"))
        open(os.path.join(d, "csrc", "t.cu"), "w").write(src)
        PKG = d
        try:
            found = _legacy_calls()
        finally:
            PKG = saved
    assert found == {("t.cu", "f", "<<<>>>"), ("t.cu", "f", "pack_weight"), ("t.cu", "f", "pdl_launch"),
                     ("t.cu", "f", "cudaMemcpy")}, found


# ---- GPU scaffolding -------------------------------------------------------------------------------------------------
def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _cudart():
    import nvidia.cuda_runtime as cr   # the CUDA runtime the torch wheel ships
    cands = [os.path.join(p, "lib", "libcudart.so.12") for p in cr.__path__]
    path = next((c for c in cands if os.path.exists(c)), None)
    assert path, cands
    return ctypes.CDLL(path)


@pytest.fixture(scope="module")
def streams():
    """Two streams created with cudaStreamNonBlocking (not torch's pool streams, whose flags are not ours to rely on)."""
    dev = _dev()
    torch.zeros(1, device=dev)
    assert torch.cuda.default_stream().cuda_stream == 0, "the default stream must be the legacy stream"
    rt = _cudart()
    rt.cudaStreamCreateWithFlags.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_uint]
    rt.cudaStreamDestroy.argtypes = [ctypes.c_void_p]
    handles, out = [], []
    for _ in range(2):
        h = ctypes.c_void_p()
        assert rt.cudaStreamCreateWithFlags(ctypes.byref(h), 1) == 0   # cudaStreamNonBlocking
        handles.append(h)
        out.append(torch.cuda.ExternalStream(h.value, device=dev))
    yield out
    torch.cuda.synchronize()
    for h in handles:
        rt.cudaStreamDestroy(h)


_CYCLES_PER_MS = []


def stall(stream, ms):
    """Enqueue a sleep of `ms` milliseconds on `stream`; returns an event recorded right after it."""
    assert 20 <= ms <= 150
    if not _CYCLES_PER_MS:
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        torch.cuda._sleep(2000000)
        b.record()
        b.synchronize()
        _CYCLES_PER_MS.append(2000000 / a.elapsed_time(b))
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(_CYCLES_PER_MS[0] * ms))
        ev = torch.cuda.Event()
        ev.record(stream)
    return ev


def _same(got, ref, what=""):
    assert len(got) == len(ref)
    for i, (g, r) in enumerate(zip(got, ref)):
        if isinstance(r, np.ndarray):
            assert np.array_equal(g, r), "%s output %d differs" % (what, i)
        elif isinstance(r, torch.Tensor):
            assert g.dtype == r.dtype and g.shape == r.shape
            assert torch.equal(g, r), "%s output %d differs: max|d| %s" % (
                what, i, (g.double() - r.double()).abs().max().item())
        else:
            assert g == r, "%s output %d differs: %r vs %r" % (what, i, g, r)


def _twice(fn, what):
    """fn() on the legacy stream, twice, with the device drained around each run; the bits must agree."""
    res = []
    for _ in range(2):
        torch.cuda.synchronize()
        out = fn()
        torch.cuda.synchronize()
        res.append(out)
    _same(res[1], res[0], what + " (reference run twice)")
    return res[0]


P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
S = lambda st: ctypes.c_void_p(st)


def _rand(g, *shape, lo=-1.0, hi=1.0):
    return (torch.rand(*shape, generator=g) * (hi - lo) + lo)


class Env:
    """The models and contexts the cases run on (built once per module)."""

    def __init__(self, dev):
        import irsde_b200 as lib
        from oracle import irsde_oracle as O
        self.lib, self.L, self.dev = lib, lib._lib, dev
        self.T = 5
        Pw = O.make_weights(3, 3, 16, 2, seed=1)
        self.nets, self.sdes, self.ctx = {}, {}, {}
        for prec in ("bf16", "fp32"):
            net = lib.ConditionalUNet(3, 3, 16, depth=2, precision=prec)
            net.load_state_dict(Pw, strict=True)
            net = net.to(dev)
            sde = lib.IRSDE(10, self.T, schedule="cosine", eps=0.005, device=dev)
            sde.set_model(net)
            self.ctx[prec] = sde._ctx_for(torch.zeros(1, device=dev))   # weights and schedule uploaded
            self.nets[prec], self.sdes[prec] = net, sde
        ae = lib.UNet(in_ch=3, out_ch=3, ch=8, ch_mult=[1, 2], embed_dim=4, precision="fp32")
        ae.load_state_dict(O.make_latent_unet_weights(3, 3, 8, [1, 2], 4, seed=2), strict=True)
        self.ae = ae.to(dev)
        self.ctx["ae"] = self.ae.sync_weights(dev)
        # a context for the standalone operator entries
        self.ctx["op"] = self.L.Context(3, 3, 8, 2, self.L.NET_CONDITIONAL, self.L.PREC_FP32, 0)

    def cuda(self, *ts):
        return [t.to(self.dev) for t in ts]


@pytest.fixture(scope="module")
def env():
    return Env(_dev())


def _pair(make):
    """(good, alt): the same inputs drawn from two generators."""
    return make(torch.Generator().manual_seed(11)), make(torch.Generator().manual_seed(22))


# ---- cases: one per stream entry (or a pair that only works together) ------------------------------------------------
B, H, W = 2, 16, 16


def _net_case(prec):
    def build(e):
        ctx = e.ctx[prec]
        good, alt = _pair(lambda g: e.cuda(_rand(g, B, 3, H, W, lo=0, hi=1), _rand(g, B, 3, H, W, lo=0, hi=1)))
        times = (ctypes.c_float * 2)(3.0, 4.0)
        outs = lambda b: [torch.full((B, 3, H, W), 7.0, device=e.dev)]
        call = lambda b, o, st: e.L.check(e.L.load().irsde_noise_fn(ctx.h, P(b[0]), P(b[1]), times, 2, P(o[0]), B, H, W, S(st)),
                                          ctx.h)
        return good, alt, outs, call
    return build


case("noise_fn_bf16", ["irsde_noise_fn"])(_net_case("bf16"))
case("noise_fn_fp32", ["irsde_noise_fn"])(_net_case("fp32"))


def _reverse_case(prec, mode, with_z, graph):
    def build(e):
        ctx, T = e.ctx[prec], e.T
        def make(g):
            ts = [_rand(g, B, 3, H, W, lo=0, hi=1), _rand(g, B, 3, H, W, lo=0, hi=1)]
            if with_z:
                ts.append(torch.randn(T, B, 3, H, W, generator=g))
            return e.cuda(*ts)
        good, alt = _pair(make)
        outs = lambda b: [torch.full((B, 3, H, W), 7.0, device=e.dev)]

        def call(b, o, st):
            L = e.L.load()
            e.L.check(L.irsde_set_image_base(ctx.h, 0), ctx.h)
            e.L.check(L.irsde_reverse(ctx.h, mode, P(b[0]), P(b[1]), P(b[2]) if with_z else None, P(o[0]), B, H, W, T, 5,
                                      1 if graph else 0, S(st)), ctx.h)
        return good, alt, outs, call
    return build


case("reverse_graph_z_bf16", ["irsde_reverse"])(_reverse_case("bf16", 0, True, True))
case("reverse_eager_philox_fp32", ["irsde_reverse"])(_reverse_case("fp32", 2, False, False))
case("reverse_graph_ode_fp32", ["irsde_reverse"])(_reverse_case("fp32", 1, False, True))


@case("trace_forward_bf16", ["irsde_trace_forward"])
def _trace(e):
    ctx, net = e.ctx["bf16"], e.nets["bf16"]
    ops = net.plan_ops(B, H, W, e.dev)
    op = [i for i, o in enumerate(ops) if o[1] is not None][len(ops) // 3]
    C_, H_, W_ = ops[op][1]
    good, alt = _pair(lambda g: e.cuda(_rand(g, B, 3, H, W, lo=0, hi=1), _rand(g, B, 3, H, W, lo=0, hi=1)))
    times = (ctypes.c_float * 1)(2.0)
    outs = lambda b: [torch.full((B, C_, H_, W_), 7.0, device=e.dev)]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_trace_forward(ctx.h, P(b[0]), P(b[1]), times, 1, B, H, W, op, P(o[0]),
                                                                     S(st)), ctx.h)
    return good, alt, outs, call


@case("latent_encode_decode", ["irsde_latent_encode", "irsde_latent_decode"])
def _latent(e):
    ctx = e.ctx["ae"]
    good, alt = _pair(lambda g: e.cuda(_rand(g, 1, 3, H, W, lo=0, hi=1), _rand(g, 1, 4, H // 2, W // 2)))
    outs = lambda b: [torch.full((1, 4, H // 2, W // 2), 7.0, device=e.dev), torch.full((1, 3, H, W), 7.0, device=e.dev)]

    def call(b, o, st):
        L = e.L.load()
        e.L.check(L.irsde_latent_encode(ctx.h, P(b[0]), P(o[0]), 1, H, W, S(st)), ctx.h)
        e.L.check(L.irsde_latent_decode(ctx.h, P(b[1]), P(o[1]), 1, H, W, S(st)), ctx.h)
    return good, alt, outs, call


@case("noise_state", ["irsde_noise_state"])
def _noise_state(e):
    ctx = e.ctx["fp32"]
    good, alt = _pair(lambda g: e.cuda(_rand(g, B, 3, H, W)))
    outs = lambda b: [torch.full((B, 3, H, W), 7.0, device=e.dev)]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_noise_state(ctx.h, P(b[0]), P(o[0]), b[0].numel(), 9, S(st)), ctx.h)
    return good, alt, outs, call


@case("uids_noise_state_images", ["irsde_set_image_uids", "irsde_noise_state_images"])
def _uids(e):
    ctx = e.ctx["fp32"]
    good, alt = _pair(lambda g: e.cuda(_rand(g, B, 3, H, W)))
    outs = lambda b: [torch.full((B, 3, H, W), 7.0, device=e.dev)]

    def call(b, o, st):
        L = e.L.load()
        e.L.check(L.irsde_set_image_uids(ctx.h, (ctypes.c_uint64 * B)(41, 17), B, S(st)), ctx.h)
        e.L.check(L.irsde_noise_state_images(ctx.h, P(b[0]), P(o[0]), B, 3 * H * W, 9, S(st)), ctx.h)
        e.L.check(L.irsde_set_image_base(ctx.h, 0), ctx.h)
    return good, alt, outs, call


@case("step", ["irsde_step"])
def _step(e):
    ctx = e.ctx["fp32"]
    good, alt = _pair(lambda g: e.cuda(*[_rand(g, B, 3, H, W) for _ in range(4)]))
    outs = lambda b: [torch.full((B, 3, H, W), 7.0, device=e.dev)]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_step(ctx.h, 0, P(b[0]), P(b[1]), P(b[2]), P(b[3]), 3, P(o[0]), b[0].numel(),
                                                            S(st)), ctx.h)
    return good, alt, outs, call


@case("step_philox", ["irsde_step_philox"])
def _step_philox(e):
    ctx = e.ctx["fp32"]
    good, alt = _pair(lambda g: e.cuda(*[_rand(g, B, 3, H, W) for _ in range(3)]))
    outs = lambda b: [torch.full((B, 3, H, W), 7.0, device=e.dev)]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_step_philox(ctx.h, 2, P(b[0]), P(b[1]), P(b[2]), 3, P(o[0]), B, 3 * H * W,
                                                                   7, S(st)), ctx.h)
    return good, alt, outs, call


@case("random_states", ["irsde_random_states"])
def _random_states(e):
    good, alt = _pair(lambda g: e.cuda(*[_rand(g, B, 3, H, W) for _ in range(3)], _rand(g, B, lo=0.1, hi=1),
                                       _rand(g, B, lo=0.1, hi=1)))
    outs = lambda b: [torch.full((B, 3, H, W), 7.0, device=e.dev)]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_random_states(P(b[0]), P(b[1]), P(b[2]), P(b[3]), P(b[4]), P(o[0]), B,
                                                                     3 * H * W, S(st)))
    return good, alt, outs, call


def _u8(g, *shape):
    return (torch.rand(*shape, generator=g) * 255.99).to(torch.uint8)


@case("img2tensor", ["irsde_img2tensor_u8"])
def _img2tensor(e):
    good, alt = _pair(lambda g: e.cuda(_u8(g, B, H, W, 3)))
    outs = lambda b: [torch.full((B, 3, H, W), 7.0, device=e.dev)]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_img2tensor_u8(P(b[0]), P(o[0]), B, 3, H, W, S(st)))
    return good, alt, outs, call


@case("tensor2img", ["irsde_tensor2img_u8"])
def _tensor2img(e):
    good, alt = _pair(lambda g: e.cuda(_rand(g, B, 3, H, W, lo=-0.1, hi=1.1)))
    outs = lambda b: [torch.full((B, H, W, 3), 7, dtype=torch.uint8, device=e.dev)]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_tensor2img_u8(P(b[0]), P(o[0]), B, 3, H, W, ctypes.c_double(0.0),
                                                                     ctypes.c_double(1.0), S(st)))
    return good, alt, outs, call


@case("sqerr_ssim", ["irsde_sqerr_u8", "irsde_ssim_u8"])
def _metrics(e):
    L = e.L.load()
    good, alt = _pair(lambda g: e.cuda(_u8(g, B, H, W, 3), _u8(g, B, H, W, 3)))
    nws = L.irsde_ssim_workspace(B, H, W, 3, 1)
    assert nws > 0
    outs = lambda b: [torch.full((B,), 7, dtype=torch.int64, device=e.dev), torch.full((nws,), 7.0, dtype=torch.float64, device=e.dev),
                      torch.full((B,), 7.0, dtype=torch.float64, device=e.dev)]

    def call(b, o, st):
        e.L.check(L.irsde_sqerr_u8(P(b[0]), P(b[1]), B, H, W, 3, 1, P(o[0]), S(st)))
        e.L.check(L.irsde_ssim_u8(P(b[0]), P(b[1]), B, H, W, 3, 1, P(o[1]), P(o[2]), S(st)))
    return good, alt, outs, call


# standalone operator entries: they wait for their stream and free their scratch (which waits for the device)
@case("conv2d_simt", ["irsde_conv2d"], hot=False)
def _conv2d(e):
    ctx = e.ctx["op"]
    good, alt = _pair(lambda g: e.cuda(_rand(g, 1, 8, 12, 12), _rand(g, 16, 8, 3, 3, lo=-0.3, hi=0.3), _rand(g, 16)))
    outs = lambda b: [torch.full((1, 16, 12, 12), 7.0, device=e.dev)]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_conv2d(ctx.h, 0, P(b[0]), P(b[1]), P(b[2]), P(o[0]), 1, 8, 12, 12, 16, 3, 3,
                                                              1, 1, 0, 1, S(st)), ctx.h)
    return good, alt, outs, call


@case("conv2d_ex_bf16_residual", ["irsde_conv2d_ex"], hot=False)
def _conv2d_ex(e):
    ctx = e.ctx["op"]
    good, alt = _pair(lambda g: e.cuda(_rand(g, 1, 16, 12, 12), _rand(g, 16, 16, 3, 3, lo=-0.2, hi=0.2), _rand(g, 16),
                                       _rand(g, 1, 16, 12, 12)))
    outs = lambda b: [torch.full((1, 16, 12, 12), 7.0, device=e.dev)]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_conv2d_ex(ctx.h, 1, P(b[0]), P(b[1]), P(b[2]), P(b[3]), P(o[0]), 1, 16, 12,
                                                                 12, 16, 3, 3, 1, 1, 0, 0, 0, S(st)), ctx.h)
    return good, alt, outs, call


@case("conv2d_fused_simt", ["irsde_conv2d_fused"], hot=False)
def _conv2d_fused(e):
    ctx = e.ctx["op"]
    good, alt = _pair(lambda g: e.cuda(_rand(g, 1, 12, 12, 16), _rand(g, 16, 16, 3, 3, lo=-0.2, hi=0.2), _rand(g, 16),
                                       _rand(g, 1, 12, 12, 16)))
    outs = lambda b: [b[3]]   # y is read and written

    def call(b, o, st):
        ep = e.L.ConvEpilogue()
        ep.bias = b[2].data_ptr()
        ep.in_pitch, ep.out_pitch = 16, 16
        e.L.check(e.L.load().irsde_conv2d_fused(ctx.h, 0, P(b[0]), P(b[1]), ctypes.byref(ep), P(b[3]), 1, 16, 12, 12, 16, 3, 3, 1, 1,
                                                0, None, S(st)), ctx.h)
    return good, alt, outs, call


@case("layernorm", ["irsde_layernorm"], hot=False)
def _layernorm(e):
    ctx = e.ctx["op"]
    good, alt = _pair(lambda g: e.cuda(_rand(g, 128, 32), _rand(g, 32, lo=0.5, hi=1.5), _rand(g, 128, 32)))
    outs = lambda b: [b[2]]

    def call(b, o, st):
        a = e.L.LnArgs()
        a.g = b[1].data_ptr()
        a.in_pitch, a.out_pitch = 32, 32
        e.L.check(e.L.load().irsde_layernorm(ctx.h, 0, P(b[0]), ctypes.byref(a), P(b[2]), 2, 64, 32, None, S(st)), ctx.h)
    return good, alt, outs, call


@case("attention_full", ["irsde_attention"], hot=False)
def _attention(e):
    ctx = e.ctx["op"]
    good, alt = _pair(lambda g: e.cuda(_rand(g, 128, 384), _rand(g, 128, 128)))
    outs = lambda b: [b[1]]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_attention(ctx.h, 0, e.L.ATTN_FULL, P(b[0]), 384, 0, P(b[1]), 128, 0, None, 0,
                                                                 None, 2, 64, None, S(st)), ctx.h)
    return good, alt, outs, call


@case("linattn_block", ["irsde_linattn_block"], hot=False)
def _linattn(e):
    ctx = e.ctx["op"]
    C, N = 64, 256
    good, alt = _pair(lambda g: e.cuda(_rand(g, N, C), _rand(g, N, C), _rand(g, C, lo=0.5, hi=1.5), _rand(g, 384, C, lo=-0.2, hi=0.2),
                                       _rand(g, C, 128, lo=-0.2, hi=0.2), _rand(g, C), _rand(g, C, lo=0.5, hi=1.5)))
    outs = lambda b: [b[1]]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_linattn_block(ctx.h, P(b[0]), C, 0, P(b[1]), C, 0, P(b[2]), P(b[3]), P(b[4]),
                                                                     P(b[5]), P(b[6]), None, 1, N, C, S(st)), ctx.h)
    return good, alt, outs, call


@case("nafnet_op_add", ["irsde_nafnet_op"], hot=False)
def _nafnet_op(e):
    ctx = e.ctx["op"]
    good, alt = _pair(lambda g: e.cuda(_rand(g, 64, 16), _rand(g, 64, 16), _rand(g, 64, 16)))
    outs = lambda b: [b[2]]

    def call(b, o, st):
        a = e.L.NafArgs()
        a.x, a.y, a.out = b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr()
        a.x_pitch = a.y_pitch = a.out_pitch = 16
        e.L.check(e.L.load().irsde_nafnet_op(ctx.h, 0, e.L.NAF_ADD, ctypes.byref(a), 1, 8, 8, 16, None, S(st)), ctx.h)
    return good, alt, outs, call


@case("time_embedding", ["irsde_time_embedding"], hot=False)
def _time_embedding(e):
    w, Sx, rows = 8, 24, 3
    good, alt = _pair(lambda g: e.cuda(_rand(g, rows, lo=0, hi=50), _rand(g, 4 * w, w), _rand(g, 4 * w), _rand(g, 4 * w, 4 * w, lo=-0.3,
                                       hi=0.3), _rand(g, 4 * w), _rand(g, Sx, 4 * w, lo=-0.3, hi=0.3), _rand(g, Sx)))
    outs = lambda b: [torch.full((rows, 4 * w), 7.0, device=e.dev), torch.full((rows, Sx), 7.0, device=e.dev)]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_time_embedding(0, P(b[0]), rows, w, P(b[1]), P(b[2]), P(b[3]), P(b[4]), P(b[5]),
                                                                      P(b[6]), Sx, P(o[0]), P(o[1]), S(st)))
    return good, alt, outs, call


@case("prep_input", ["irsde_prep_input"], hot=False)
def _prep_input(e):
    good, alt = _pair(lambda g: e.cuda(_rand(g, 1, 3, 8, 8), _rand(g, 1, 3, 8, 8), _rand(g, 1, 8, 8, 8)))
    outs = lambda b: [b[2]]
    call = lambda b, o, st: e.L.check(e.L.load().irsde_prep_input(0, P(b[0]), P(b[1]), P(b[2]), 1, 3, 8, 8, 8, 8, 8, 1, 1, 0, 0, 0, 0,
                                                                  S(st)))
    return good, alt, outs, call


def _reference(e, name):
    good, alt, outs, call = CASES[name][0](e)

    def run():
        bufs = [t.clone() for t in good]
        o = outs(bufs)
        call(bufs, o, 0)
        return [t.clone() for t in o]
    return good, alt, outs, call, _twice(run, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_s1_producer_on_the_callers_stream(env, streams, name):
    s = streams[0]
    good, alt, outs, call, ref = _reference(env, name)
    bufs = [t.clone() for t in alt]      # a different valid input until the producer on s overwrites it
    o = outs(bufs)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        stall(s, 100)
        for b, g in zip(bufs, good):
            b.copy_(g)
        call(bufs, o, s.cuda_stream)
        got = [t.clone() for t in o]
    torch.cuda.synchronize()
    _same(got, ref, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_s2_no_legacy_stream_work_when_warm(env, streams, name):
    s = streams[0]
    good, alt, outs, call, ref = _reference(env, name)   # also warms plans, graphs and kernels
    bufs = [t.clone() for t in good]
    o = outs(bufs)
    torch.cuda.synchronize()
    legacy = stall(torch.cuda.default_stream(), 150)
    pending = stall(s, 60)
    with torch.cuda.stream(s):
        call(bufs, o, s.cuda_stream)
        got = [t.clone() for t in o]
    if CASES[name][2]:
        assert not pending.query(), "%s returned only after its stream drained" % name
        s.synchronize()
        assert not legacy.query(), "%s made its stream wait for the legacy stream" % name
    torch.cuda.synchronize()
    _same(got, ref, name)


# ---- S3: cold calls with the legacy stream stalled --------------------------------------------------------------------
def _fresh_unet(prec, nf=16, T=5):
    import irsde_b200 as lib
    from oracle import irsde_oracle as O
    dev = _dev()
    net = lib.ConditionalUNet(3, 3, nf, depth=2, precision=prec)
    net.load_state_dict(O.make_weights(3, 3, nf, 2, seed=4), strict=True)
    net = net.to(dev)
    sde = lib.IRSDE(10, T, schedule="cosine", eps=0.005, device=dev)
    sde.set_model(net)
    sde._ctx_for(torch.zeros(1, device=dev))   # weights and schedule uploaded: only the plan is cold
    torch.cuda.synchronize()
    return net, sde


def _fresh_naf():
    import irsde_b200 as lib
    from oracle import irsde_oracle as O
    net = lib.ConditionalNAFNet(img_channel=3, width=16, middle_blk_num=1, enc_blk_nums=[1], dec_blk_nums=[1], precision="bf16")
    net.load_state_dict(O.make_nafnet_weights(3, 16, 1, [1], [1], seed=3), strict=True)
    net = net.to(_dev())
    net.sync_weights(_dev())
    return net


def _fresh_ae():
    import irsde_b200 as lib
    from oracle import irsde_oracle as O
    ae = lib.UNet(in_ch=3, out_ch=3, ch=8, ch_mult=[1, 2], embed_dim=4, precision="bf16")
    ae.load_state_dict(O.make_latent_unet_weights(3, 3, 8, [1, 2], 4, seed=2), strict=True)
    ae = ae.to(_dev())
    ae.sync_weights(_dev())
    return ae


def _s3_inputs(shape):
    g = torch.Generator().manual_seed(5)
    return [t.to(_dev()) for t in (torch.rand(*shape, generator=g), torch.rand(*shape, generator=g))]


def _s3_run(kind, stream):
    """Build fresh objects, warm what the scenario needs warm, then run the cold part on `stream` (None: legacy)."""
    shape = (1, 3, 20, 28)
    if kind in ("bf16_stem", "fp32"):
        net, _ = _fresh_unet("bf16" if kind == "bf16_stem" else "fp32")
        fn = lambda x, mu: net(x, mu, 3)
    elif kind == "nafnet":
        net = _fresh_naf()
        fn = lambda x, mu: net(x, mu, 3)
    elif kind == "latent":
        ae = _fresh_ae()
        fn = lambda x, mu: ae.decode(*ae.encode(x))
    elif kind == "graph_capture":
        net, sde = _fresh_unet("bf16")
        sde.rng, sde.seed_auto_increment = "philox", False
        x, mu = _s3_inputs(shape)
        sde.use_graph = False
        sde.set_mu(mu)
        sde.reverse_ode(x)          # the plan is warm; the first capture of the ODE graph happens below
        sde.use_graph = True
        torch.cuda.synchronize()
        fn = lambda x, mu: (sde.set_mu(mu), sde.reverse_ode(x))[1]
    else:   # chain_T150: the first chain of a warm plan grows the time table past 128 rows
        net, sde = _fresh_unet("fp32", nf=8, T=150)
        sde.rng, sde.seed_auto_increment = "philox", False
        x, mu = _s3_inputs(shape)
        net(x, mu, 3)
        torch.cuda.synchronize()
        fn = lambda x, mu: (sde.set_mu(mu), sde.reverse_sde(x))[1]
    x, mu = _s3_inputs(shape)
    torch.cuda.synchronize()
    if stream is None:
        out = fn(x, mu)
    else:
        stall(torch.cuda.default_stream(), 150)
        with torch.cuda.stream(stream):
            out = fn(x, mu).clone()
    torch.cuda.synchronize()
    return [out]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["bf16_stem", "fp32", "nafnet", "latent", "graph_capture", "chain_T150"])
def test_s3_cold_calls_with_the_legacy_stream_stalled(streams, kind):
    ref = _twice(lambda: _s3_run(kind, None), kind)
    _same(_s3_run(kind, streams[0]), ref, kind)


# ---- S4: weights produced on a stream ---------------------------------------------------------------------------------
@pytest.mark.gpu
def test_s4_load_tensor_reads_device_data_after_its_producer(streams):
    import irsde_b200 as lib
    from oracle import irsde_oracle as O
    dev, s = _dev(), streams[0]
    Pw, Palt = O.make_weights(3, 3, 8, 2, seed=6), O.make_weights(3, 3, 8, 2, seed=7)
    x, mu = _s3_inputs((1, 3, 16, 16))

    def forward(net):
        return [net(x, mu, 4)]
    ref_net = lib.ConditionalUNet(3, 3, 8, depth=2, precision="fp32")
    ref_net.load_state_dict(Pw, strict=True)
    ref_net = ref_net.to(dev)
    ref = _twice(lambda: forward(ref_net), "forward")

    net = lib.ConditionalUNet(3, 3, 8, depth=2, precision="fp32")
    net.load_state_dict(Palt, strict=True)
    net = net.to(dev)
    ctx = net.sync_weights(dev)      # finalized with the other weights: the next load starts an upload round
    L = lib._lib.load()
    names = list(Pw)
    target = names[-1]
    srcs = {n: Pw[n].to(dev).contiguous() for n in names}
    buf = Palt[target].to(dev).contiguous()   # holds other valid weights until the producer on s overwrites it
    torch.cuda.synchronize()
    for n in names[:-1]:
        t = srcs[n]
        lib._lib.check(L.irsde_load_tensor(ctx.h, n.encode(), P(t), t.dim(), (ctypes.c_int64 * t.dim())(*t.shape)), ctx.h)
    with torch.cuda.stream(s):
        stall(s, 100)
        buf.copy_(srcs[target])
    lib._lib.check(L.irsde_load_tensor(ctx.h, target.encode(), P(buf), buf.dim(), (ctypes.c_int64 * buf.dim())(*buf.shape)), ctx.h)
    lib._lib.check(L.irsde_finalize_weights(ctx.h), ctx.h)
    out = torch.empty(1, 3, 16, 16, device=dev)
    lib._lib.check(L.irsde_noise_fn(ctx.h, P(x), P(mu), (ctypes.c_float * 1)(4.0), 1, P(out), 1, 16, 16, None), ctx.h)
    torch.cuda.synchronize()
    _same([out], ref, "noise_fn after load_tensor")

    # sync_weights converts channels-last parameters on the current stream just before each upload
    net2 = lib.ConditionalUNet(3, 3, 8, depth=2, precision="fp32")
    net2.load_state_dict(Pw, strict=True)
    net2 = net2.to(dev)
    net2.plan_ops(1, 16, 16, dev)    # the plan is warm; the new parameter tensors below are uploaded again under s
    for p in net2.parameters():
        if p.dim() == 4:
            p.data = p.data.contiguous(memory_format=torch.channels_last)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        stall(s, 100)
        got = [net2(x, mu, 4).clone()]
    torch.cuda.synchronize()
    _same(got, ref, "forward after sync_weights on a stream")


# ---- S5: two streams, one context ------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_s5_image_uids_set_on_another_stream_wait_for_the_chain(env, streams):
    s1, s2 = streams
    ctx, L, T = env.ctx["fp32"], env.L.load(), env.T
    good, _ = _pair(lambda g: env.cuda(_rand(g, B, 3, H, W, lo=0, hi=1), _rand(g, B, 3, H, W, lo=0, hi=1)))
    u1, u2 = (ctypes.c_uint64 * B)(3, 8), (ctypes.c_uint64 * B)(100, 200)

    def chain(st, out):
        env.L.check(L.irsde_reverse(ctx.h, 0, P(good[0]), P(good[1]), None, P(out), B, H, W, T, 1, 1, S(st)), ctx.h)

    def noise(st, out):
        env.L.check(L.irsde_noise_state_images(ctx.h, P(good[1]), P(out), B, 3 * H * W, 2, S(st)), ctx.h)

    def ref_run():
        a, b = torch.empty(B, 3, H, W, device=env.dev), torch.empty(B, 3, H, W, device=env.dev)
        env.L.check(L.irsde_set_image_uids(ctx.h, u1, B, None), ctx.h)
        chain(0, a)
        env.L.check(L.irsde_set_image_uids(ctx.h, u2, B, None), ctx.h)
        noise(0, b)
        return [a, b]
    ref = _twice(ref_run, "uids")
    a, b = torch.full((B, 3, H, W), 7.0, device=env.dev), torch.full((B, 3, H, W), 7.0, device=env.dev)
    env.L.check(L.irsde_set_image_uids(ctx.h, u1, B, None), ctx.h)
    torch.cuda.synchronize()
    stall(s1, 100)
    chain(s1.cuda_stream, a)         # reads the uids when it runs, after the stall
    env.L.check(L.irsde_set_image_uids(ctx.h, u2, B, S(s2.cuda_stream)), ctx.h)
    noise(s2.cuda_stream, b)
    torch.cuda.synchronize()
    env.L.check(L.irsde_set_image_base(ctx.h, 0), ctx.h)
    _same([a, b], ref, "chain on s1 / uids on s2")


@pytest.mark.gpu
def test_s5_decode_on_another_stream_waits_for_encode(env, streams):
    s1, s2 = streams
    ae = env.ae
    xa, xb = _pair(lambda g: env.cuda(_rand(g, 1, 3, H, W, lo=0, hi=1)))
    xa, xb = xa[0], xb[0]

    def ref_run():
        z, h = ae.encode(xb)
        return [z, ae.decode(z, h)]
    zr, outr = _twice(ref_run, "latent")
    ae.encode(xa)                    # the skips of another image until the encode on s1 runs
    torch.cuda.synchronize()
    stall(s1, 100)
    with torch.cuda.stream(s1):
        z, h = ae.encode(xb)
    with torch.cuda.stream(s2):
        out = ae.decode(zr, h)
    torch.cuda.synchronize()
    _same([z, out], [zr, outr], "encode on s1 / decode on s2")


@pytest.mark.gpu
def test_s5_noise_fn_on_another_stream_after_a_chain(env, streams):
    s1, s2 = streams
    ctx, L, T = env.ctx["bf16"], env.L.load(), env.T
    good, _ = _pair(lambda g: env.cuda(_rand(g, B, 3, H, W, lo=0, hi=1), _rand(g, B, 3, H, W, lo=0, hi=1)))
    times = (ctypes.c_float * 1)(2.0)

    def run(st1, st2):
        a, b = torch.full((B, 3, H, W), 7.0, device=env.dev), torch.full((B, 3, H, W), 7.0, device=env.dev)
        env.L.check(L.irsde_set_image_base(ctx.h, 0), ctx.h)
        env.L.check(L.irsde_reverse(ctx.h, 0, P(good[0]), P(good[1]), None, P(a), B, H, W, T, 1, 1, S(st1)), ctx.h)
        env.L.check(L.irsde_noise_fn(ctx.h, P(good[0]), P(good[1]), times, 1, P(b), B, H, W, S(st2)), ctx.h)
        return [a, b]
    ref = _twice(lambda: run(0, 0), "chain + noise_fn")
    torch.cuda.synchronize()
    stall(s1, 100)
    got = run(s1.cuda_stream, s2.cuda_stream)
    torch.cuda.synchronize()
    _same(got, ref, "chain on s1 / noise_fn on s2")


# ---- S6: Python front-ends under torch.cuda.stream(s) -----------------------------------------------------------------
def _front(name, env):
    import irsde_b200 as lib
    from oracle import irsde_oracle as O
    dev = env.dev
    g = torch.Generator().manual_seed(3)
    X, M = torch.rand(B, 3, H, W, generator=g).to(dev), torch.rand(B, 3, H, W, generator=g).to(dev)
    U8 = (torch.rand(B, H, W, 3, generator=g) * 255.99).to(torch.uint8).to(dev)
    if name.startswith("irsde_"):
        _, mode, rng, graph = name.split("_")
        sde = env.sdes["bf16"]

        def fn():
            sde.rng, sde.use_graph, sde.seed, sde.seed_auto_increment = rng, graph == "graph", 0, False
            torch.manual_seed(0)
            x, mu = X.clone(), M.clone()
            sde.set_mu(mu)
            out = getattr(sde, "reverse_" + mode)(x)
            sde.rng, sde.use_graph = "torch", True
            return [out]
        return fn
    if name == "denoising_sde":
        net = lib.DenoisingUNet(3, 3, 16, depth=2, precision="fp32")
        net.load_state_dict(O.make_weights(3, 3, 16, 2, variant="denoising", seed=5), strict=True)
        net = net.to(dev)
        sde = lib.DenoisingSDE(10, env.T, device=dev)
        sde.set_model(net)

        def fn():
            sde.rng, sde.seed, sde.seed_auto_increment = "philox", 0, False
            return [sde.reverse_sde(X.clone()), sde.reverse_ode(X.clone())]
        return fn
    if name == "nafnet":
        net = _fresh_naf()
        return lambda: [net(X.clone(), M.clone(), 3)]
    if name == "unet_encode_decode":
        ae = env.ae
        return lambda: (lambda z, h: [z, ae.decode(z.clone(), h)])(*ae.encode(X[:1].clone()))
    if name == "tiled_refusion":
        ae = lib.UNet(in_ch=3, out_ch=3, ch=8, ch_mult=[1, 2], embed_dim=4, precision="fp32")
        ae.load_state_dict(O.make_latent_unet_weights(3, 3, 8, [1, 2], 4, seed=2), strict=True)
        ae = ae.to(dev)
        net = lib.ConditionalNAFNet(img_channel=4, width=16, middle_blk_num=1, enc_blk_nums=[1, 1], dec_blk_nums=[1, 1], latent=True,
                                    precision="fp32")
        net.load_state_dict(O.make_nafnet_weights(4, 16, 1, [1, 1], [1, 1], seed=3), strict=True)
        net = net.to(dev)
        sde = lib.IRSDE(50, 3, schedule="cosine", eps=0.005, device=dev)
        sde.set_model(net)
        pipe = lib.TiledRefusion(ae, sde, tile=8, mode="sde", seed=5)
        Xr = torch.rand(1, 3, 32, 32, generator=g).to(dev)
        return lambda: [pipe.restore(Xr.clone())[0]]
    if name == "imaging":
        im = lib.imaging

        def fn():
            a, b = U8.clone(), U8.flip(1).contiguous()
            t = im.img2tensor_device(a)
            return [t, im.tensor2img_device(t * 0.9), im.calculate_psnr(a[0], b[0]), im.calculate_ssim(a[0], b[0])]
        return fn
    raise KeyError(name)


FRONT_ENDS = ["irsde_sde_philox_graph", "irsde_ode_torch_eager", "irsde_posterior_torch_graph", "irsde_sde_torch_eager",
              "denoising_sde", "nafnet", "unet_encode_decode", "tiled_refusion", "imaging"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", FRONT_ENDS)
def test_s6_front_ends_under_a_stream(env, streams, name):
    s = streams[0]
    fn = _front(name, env)
    ref = _twice(fn, name)
    with torch.cuda.stream(s):
        stall(s, 80)
        got = fn()
        got = [t.clone() if isinstance(t, torch.Tensor) else t for t in got]
    torch.cuda.synchronize()
    _same(got, ref, name)


@pytest.mark.gpu
def test_s6_restorer_with_its_main_stream_stalled(env, streams):
    import irsde_b200 as lib
    s = streams[0]
    rng = np.random.RandomState(4)
    images = [(rng.rand(16, 16, 3) * 255).astype(np.uint8) for _ in range(6)] + \
             [(rng.rand(20, 12, 3) * 255).astype(np.uint8) for _ in range(2)]
    r = lib.Restorer(env.sdes["fp32"], mode="sde", batch_size=2, seed=3)
    ref = _twice(lambda: r.restore(images), "Restorer")      # also warms both plans
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        stall(s, 100)
        got = r.restore(images)
    torch.cuda.synchronize()
    _same(got, ref, "Restorer")
