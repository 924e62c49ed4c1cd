#!/usr/bin/env python
"""Per-launch timing of every tap-GEMM conv of the c2 sampler step (ConditionalUNet nf=64 depth=4, 8x3x256x256, bf16).

Runs a few sampler steps in eager mode (no graph replay) with CUDA events around every plan op and prints, for each conv
op: its label, the conv_tc_persist_kernel<BN, MODE, EKT> it runs, its output tiles, ms per sampler step and the TFLOP/s
implied by the plan's FLOP count; then totals per (BN, MODE) class.  A second, separate pass of one step with
IRSDE_TC_DEBUG=1 supplies the kernel of each launch and its cycle counters (producer waits on empty barriers, each
consumer warpgroup's waits on full barriers, epilogue cycles and ping-pong turn waits); that pass synchronizes after
every conv, so its times are not used.

  python scripts/profile_convs.py [--steps 5] [--json OUT]

IRSDE_B200_LIB selects another build of the library (A/B runs).
"""
import argparse
import collections
import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CATS = ["wgmma_conv", "simt_conv", "layernorm", "attention", "misc", "update"]
MODE_NAME = {0: "per-tap", 2: "ROWS", 3: "fp32x3"}
TCDBG = re.compile(r"TCDBG BN=(\d+) mode=(\d+) ekt=(\d+) grid=(\d+) tiles=(\d+) .*\| prod wait (\S+) / (\S+) \| "
                   r"wg0 full (\S+) epi (\S+) turn (\S+) / (\S+) \(tiles/cta (\S+)\) \| "
                   r"wg1 full (\S+) epi (\S+) turn (\S+) / (\S+) \(tiles/cta (\S+)\)")
# the counter line of builds before the ping-pong schedule (one record for both consumer warpgroups, no EKT)
TCDBG_COOP = re.compile(r"TCDBG BN=(\d+) mode=(\d+) grid=(\d+) tiles=(\d+) .*\| prod wait (\S+) / (\S+) \| "
                        r"consumer wait full (\S+) / (\S+) \(tiles/cta (\S+)\)")


def tcdbg(line):
    """The counters of one TCDBG line in the current layout (older builds: EKT -1, no epilogue / turn counters)."""
    m = TCDBG.search(line)
    if m:
        return [float(x) for x in m.groups()]
    m = TCDBG_COOP.search(line)
    if m:
        bn, mode, grid, tiles, pw, pt, full, tot, tpc = [float(x) for x in m.groups()]
        return [bn, mode, -1, grid, tiles, pw, pt, full, 0, 0, tot, tpc, 0, 0, 0, 0, 0]
    return None


def wg_shares(c):
    """One consumer warpgroup's counters (full wait, epilogue, turn wait, cycles, tiles per CTA) as shares of its cycles."""
    full, epi, turn, total, tpc = c
    f = 1.0 / total if total else 0.0
    return {"full": full * f, "epi": epi * f, "turn": turn * f, "tiles_per_cta": tpc}


def captured_stderr(fn):
    """Run fn() with fd 2 redirected to a temporary file; return its lines (the library writes PROF / TCDBG there)."""
    with tempfile.TemporaryFile(mode="w+") as tf:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(tf.fileno(), 2)
        try:
            fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tf.seek(0)
        return tf.read().splitlines()


def prof_ops(lines):
    """[(label, ms, flops)] of the wgmma_conv PROF lines, in launch order."""
    out = []
    for line in lines:
        f = line.split("\t")
        if len(f) < 6 or f[0] != "PROF" or int(f[1]) != CATS.index("wgmma_conv"):
            continue
        ms, tflops = float(f[2]), float(f[3])
        out.append((f[5], ms, tflops * 1e12 * ms * 1e-3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="sampler steps in the timed pass")
    ap.add_argument("--json", help="also write the result as JSON to this file")
    args = ap.parse_args()

    import torch
    import irsde_b200
    from irsde_b200 import _lib

    if not torch.cuda.is_available():
        raise SystemExit("profile_convs.py: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = irsde_b200.ConditionalUNet(3, 3, 64, depth=4, precision="bf16").to(dev)
    sde = irsde_b200.IRSDE(10, 100, schedule="cosine", eps=0.005, device=dev)
    sde.set_model(net)
    sde.use_graph = False
    sde.rng = "philox"
    g = torch.Generator().manual_seed(1234)
    lq = torch.rand(8, 3, 256, 256, generator=g)
    xT = (lq + torch.randn(lq.shape, generator=g) * 10).to(dev)
    sde.set_mu(lq.to(dev))
    ctx = net.sync_weights(dev)
    sde.reverse_sde(xT, T=2)  # warm-up: plan, descriptors, first-launch module loads
    torch.cuda.synchronize()

    ncat = len(CATS)
    ms_a, fl_a, n_a, by_a = ((ctypes.c_double * ncat)(), (ctypes.c_double * ncat)(), (ctypes.c_int64 * ncat)(),
                             (ctypes.c_double * ncat)())

    def profiled(steps):
        def run():
            _lib.check(ctx.L.irsde_profile_begin(ctx.h), ctx.h)
            sde.reverse_sde(xT, T=steps)
            _lib.check(ctx.L.irsde_profile_end_bytes(ctx.h, ms_a, fl_a, n_a, by_a, ncat), ctx.h)
        return run

    os.environ["IRSDE_PROFILE_DUMP"] = "1"
    # pass 1 (timed): PROF lines only
    timed = prof_ops(captured_stderr(profiled(args.steps)))
    conv_ms = ms_a[CATS.index("wgmma_conv")] / args.steps
    # pass 2 (one step, counters on): the kernel and counters of every conv launch, matched to the ops in launch order
    os.environ["IRSDE_TC_DEBUG"] = "1"
    try:
        lines = captured_stderr(profiled(1))
    finally:
        del os.environ["IRSDE_TC_DEBUG"]
    dbg = [d for d in map(tcdbg, lines) if d]
    ops_one = prof_ops(lines)
    if len(dbg) != len(ops_one) or len(timed) != len(ops_one) * args.steps:
        raise SystemExit("profile_convs.py: %d conv launches with counters, %d conv ops per step, %d timed launches over %d steps"
                         % (len(dbg), len(ops_one), len(timed), args.steps))

    per = len(ops_one)
    rows = collections.OrderedDict()
    for i, (label, ms, fl) in enumerate(timed):
        d = dbg[i % per]
        assert label == ops_one[i % per][0], (label, ops_one[i % per][0])
        key = (i % per, label)
        r = rows.setdefault(key, {"label": label, "bn": int(d[0]), "mode": int(d[1]), "ekt": int(d[2]), "tiles": int(d[4]),
                                  "grid": int(d[3]), "ms": 0.0, "flops": 0.0,
                                  "prod_wait": d[5] / d[6] if d[6] else 0.0,
                                  "wg": [wg_shares(d[7 + 5 * w:12 + 5 * w]) for w in (0, 1)]})
        r["ms"] += ms / args.steps
        r["flops"] = fl
    out = {"gpu": torch.cuda.get_device_name(0), "steps": args.steps, "conv_ms_per_step": conv_ms, "ops": list(rows.values())}
    try:
        out["power_limit_max_sm_clock"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm",
                                                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except Exception:
        out["power_limit_max_sm_clock"] = None

    print("%-44s %-16s %6s %8s %7s | %5s | %s" % ("conv op (weight label)", "<BN,MODE,EKT>", "tiles", "ms/step", "TFLOP/s",
                                                  "prod", "share of cycles per warpgroup: full wait / epilogue / turn wait"))
    classes = collections.OrderedDict()
    for r in out["ops"]:
        tf = r["flops"] / (r["ms"] * 1e-3) / 1e12 if r["ms"] > 0 else 0.0
        r["tflops"] = tf
        wgs = "  ".join("wg%d %3.0f%% %3.0f%% %3.0f%%" % (w, 100 * x["full"], 100 * x["epi"], 100 * x["turn"])
                        for w, x in enumerate(r["wg"]) if x["tiles_per_cta"] > 0)
        print("%-44s %-16s %6d %8.4f %7.0f | %4.0f%% | %s" % (r["label"][:44], "<%d,%d,%d>" % (r["bn"], r["mode"], r["ekt"]),
                                                             r["tiles"], r["ms"], tf, 100 * r["prod_wait"], wgs))
        c = classes.setdefault("%s BN=%d" % (MODE_NAME.get(r["mode"], str(r["mode"])), r["bn"]), {"ms": 0.0, "flops": 0.0, "ops": 0})
        c["ms"] += r["ms"]
        c["flops"] += r["flops"]
        c["ops"] += 1
    print()
    for k, c in classes.items():
        c["tflops"] = c["flops"] / (c["ms"] * 1e-3) / 1e12 if c["ms"] > 0 else 0.0
        print("class %-14s %3d ops  %7.3f ms/step  %5.0f TFLOP/s" % (k, c["ops"], c["ms"], c["tflops"]))
    out["classes"] = classes
    print("all tap-GEMM convs: %.3f ms/step" % conv_ms)
    print("GPU: %s, power limit / max SM clock: %s" % (out["gpu"], out["power_limit_max_sm_clock"]))
    if args.json:
        with open(args.json, "w") as fjson:
            json.dump(out, fjson, indent=1)


if __name__ == "__main__":
    main()
