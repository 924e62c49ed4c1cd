#!/usr/bin/env python
"""Per-launch timing of every attention block of the c2 sampler step (ConditionalUNet nf=64 depth=4, 8x3x256x256, bf16).

Runs a few sampler steps in eager mode (no graph replay) with CUDA events around every plan op, then prints, for each
Residual(PreNorm(LinearAttention)) block, the time of each of its ops per sampler step, its algorithmic bytes and the
rate those bytes imply, and the layernorm / attention category totals.

  python scripts/profile_attention.py [--steps 5] [--json OUT]

IRSDE_B200_LIB selects another build of the library (A/B runs).
"""
import argparse
import collections
import ctypes
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BLOCK = re.compile(r"^((?:downs|ups)\.\d+\.2\.|mid_attn\.)")
CATS = ["wgmma_conv", "simt_conv", "layernorm", "attention", "misc", "update"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="sampler steps in the instrumented pass")
    ap.add_argument("--json", help="also write the result as JSON to this file")
    args = ap.parse_args()

    import torch
    import irsde_b200
    from irsde_b200 import _lib

    if not torch.cuda.is_available():
        raise SystemExit("profile_attention.py: needs a CUDA device")
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
    # the library prints one PROF line per op to fd 2 when IRSDE_PROFILE_DUMP=1 (read when the profile ends)
    os.environ["IRSDE_PROFILE_DUMP"] = "1"
    with tempfile.TemporaryFile(mode="w+") as tf:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(tf.fileno(), 2)
        try:
            _lib.check(ctx.L.irsde_profile_begin(ctx.h), ctx.h)
            sde.reverse_sde(xT, T=args.steps)
            _lib.check(ctx.L.irsde_profile_end_bytes(ctx.h, ms_a, fl_a, n_a, by_a, ncat), ctx.h)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tf.seek(0)
        lines = tf.read().splitlines()

    blocks = collections.OrderedDict()
    for line in lines:
        f = line.split("\t")
        if len(f) < 6 or f[0] != "PROF":
            continue
        label, ms = f[5], float(f[2])
        m = BLOCK.match(label)
        if not m:
            continue
        ops = blocks.setdefault(m.group(1), collections.OrderedDict())
        rec = ops.setdefault(label, {"ms": 0.0, "n": 0, "gbs": float(f[4])})
        rec["ms"] += ms
        rec["n"] += 1
    S = args.steps
    out = {"gpu": torch.cuda.get_device_name(0), "steps": S, "blocks": {},
           "categories": {CATS[i]: {"ms_per_step": ms_a[i] / S, "ops_per_step": n_a[i] / S} for i in range(ncat) if n_a[i] > 0}}
    try:
        import subprocess
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                            capture_output=True, text=True).stdout.strip()
    except Exception:
        out["power_limit"] = None
    total = 0.0
    for blk, ops in blocks.items():
        bms = sum(r["ms"] for r in ops.values()) / S
        total += bms
        out["blocks"][blk] = {"ms_per_step": bms, "ops": {k: {"ms_per_step": r["ms"] / S, "launch_groups_per_step": r["n"] / S,
                                                              "algorithmic_gbs": r["gbs"]} for k, r in ops.items()}}
        print("%-14s %.3f ms/step" % (blk, bms))
        for k, r in ops.items():
            print("    %-70s %8.4f ms  %7.0f GB/s" % (k[len(blk):][:70], r["ms"] / S, r["gbs"]))
    out["attention_blocks_ms_per_step"] = total
    print("all attention blocks: %.3f ms/step" % total)
    for k in ("layernorm", "attention"):
        if k in out["categories"]:
            print("category %-10s %.3f ms/step, %.0f ops/step" % (k, out["categories"][k]["ms_per_step"], out["categories"][k]["ops_per_step"]))
    print("GPU: %s, %s" % (out["gpu"], out["power_limit"]))
    if args.json:
        with open(args.json, "w") as fjson:
            json.dump(out, fjson, indent=1)


if __name__ == "__main__":
    main()
