#!/usr/bin/env python
"""Time the denoising-sde task's Refusion workload (codes/config/denoising-sde/options/test/refusion.yml) on one GPU.

DenoisingSDE(max_sigma=70, T=1000) drives DenoisingNAFNet(3, 64, 1, [1, 1, 1, 28], [1, 1, 1, 1]); test.py runs
reverse_ode from T* = get_optimal_timestep(15) = 158.  No trained checkpoint is available offline, so the weights are
random (beta / gamma set to 0.1: at the reference's zero init every NAFBlock is the identity).  Batch 1 at the Kodak size
(512 x 768) and the CBSD68 size (321 x 481, zero-padded to 336 x 496 inside the network), bf16 and fp32x3, on the
captured graph chain.  One JSON line per case:

  card, power limit and SM clock (nvidia-smi, read while the timed chains run), ms per sampler step (CUDA events over
  whole chains after a warm-up chain), img/s, launches per step, irsde_device_bytes, and max |x0(bf16) - x0(fp32x3)|.

  python scripts/bench_denoising_sde.py [--chains 2] [--reference] [--reference-steps 10]

--reference also times the reference's own classes (oracle/_ref, staged by build()) in PyTorch eager on the same GPU,
for context; it is skipped when that tree is absent.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NET = dict(img_channel=3, width=64, middle_blk_num=1, enc_blk_nums=[1, 1, 1, 28], dec_blk_nums=[1, 1, 1, 1])
SIZES = {"kodak": (512, 768), "cbsd68": (321, 481)}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [f.strip() for f in out.split(",")]
        return {"card": name, "power_limit_w": float(pl), "sm_clock_mhz": int(sm), "sm_clock_max_mhz": int(smax)}
    except Exception as e:  # the timing stays valid; the line says what could not be read
        return {"card": None, "power_limit_w": None, "sm_clock_mhz": None, "nvidia_smi": repr(e)}


def time_chains(torch, fn, n):
    """ms per chain over n chains (CUDA events) and the card's state read while they run."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        out = fn()
    e1.record()
    info = gpu_info()        # the chains are still running: this reads the clock under load
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, info, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=2, help="timed whole chains per case (after one warm-up chain)")
    ap.add_argument("--reference", action="store_true", help="also time the reference's classes in PyTorch eager")
    ap.add_argument("--reference-steps", type=int, default=10, help="sampler steps of the timed reference chain")
    args = ap.parse_args()
    import torch
    import irsde_b200
    if not torch.cuda.is_available():
        raise SystemExit("bench_denoising_sde needs a CUDA device (an H100); there is no CPU measurement")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    state = irsde_b200.DenoisingNAFNet(**NET).state_dict()
    for k, v in state.items():
        if k.endswith(("beta", "gamma")):
            v.fill_(0.1)
    sde_cfg = dict(max_sigma=70, T=1000)
    for size, (H, W) in SIZES.items():
        g = torch.Generator().manual_seed(1)
        xn = (torch.rand(1, 3, H, W, generator=g) + torch.randn(1, 3, H, W, generator=g) * (15 / 255)).to(dev)
        x0 = {}
        for precision in ("bf16", "fp32x3"):
            net = irsde_b200.DenoisingNAFNet(precision=precision, **NET)
            net.load_state_dict(state, strict=True)
            net = net.to(dev)
            sde = irsde_b200.DenoisingSDE(device=dev, **sde_cfg)
            sde.use_graph = True
            sde.set_model(net)
            T = sde.get_optimal_timestep(15)
            steps = int(T)
            with torch.no_grad():
                sde.reverse_ode(xn, T=T)               # plan, weights, graph capture
                torch.cuda.synchronize()
                l0 = net.launch_count()
                ms_chain, info, out = time_chains(torch, lambda: sde.reverse_ode(xn, T=T), args.chains)
                launches = net.launch_count() - l0
            x0[precision] = out.float()
            line = {"workload": "denoising-sde refusion.yml reverse_ode", "size": size, "batch": 1, "H": H, "W": W,
                    "precision": precision, "graph": True, "T": sde_cfg["T"], "T_star": steps,
                    "ms_per_step": ms_chain / steps, "ms_per_chain": ms_chain, "img_per_s": 1000.0 / ms_chain,
                    "launches_per_step": launches / (args.chains * steps),
                    "device_bytes": int(net._ctx.L.irsde_device_bytes(net._ctx.h)),
                    "finite": bool(torch.isfinite(out).all()), "chains_timed": args.chains}
            line.update(info)
            if precision == "fp32x3":
                line["max_abs_x0_bf16_vs_fp32x3"] = (x0["bf16"] - x0["fp32x3"]).abs().max().item()
            print(json.dumps(line), flush=True)
            del net, sde
            torch.cuda.empty_cache()
        if args.reference:
            reference(torch, dev, xn, state, sde_cfg, size, H, W, args.reference_steps)


def reference(torch, dev, xn, state, sde_cfg, size, H, W, nsteps):
    """The reference's own DenoisingSDE + denoising-sde ConditionalNAFNet in PyTorch eager (torch's default TF32 settings,
    as the reference never touches them), timed over nsteps sampler steps."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import ref_loader
    if not ref_loader.available():
        print(json.dumps({"impl": "reference", "size": size, "unavailable": "oracle/_ref not staged"}), flush=True)
        return
    utils, mods = ref_loader.load("denoising-sde")
    net = mods.ConditionalNAFNet(**NET)
    net.load_state_dict(state, strict=True)
    net = net.to(dev).eval()
    sde = utils.DenoisingSDE(device=dev, **sde_cfg)
    sde.set_model(net)
    with torch.no_grad():
        sde.reverse_ode(xn, T=2)
        torch.cuda.synchronize()
        ms, info, out = time_chains(torch, lambda: sde.reverse_ode(xn, T=nsteps), 1)
    line = {"impl": "reference", "workload": "denoising-sde refusion.yml reverse_ode", "size": size, "batch": 1, "H": H, "W": W,
            "precision": "fp32 eager (torch default TF32)", "steps_timed": nsteps, "ms_per_step": ms / nsteps,
            "img_per_s_at_T_star_158": 1000.0 / (ms / nsteps * 158), "finite": bool(torch.isfinite(out).all())}
    line.update(info)
    print(json.dumps(line), flush=True)
    del net, sde
    torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
