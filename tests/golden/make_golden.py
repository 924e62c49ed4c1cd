"""Generate golden fixtures by running the UNMODIFIED reference (imported from
/root/reference) on CPU in fp32.  Run once in the build container:

    python tests/golden/make_golden.py

The GPU box has no /root/reference; tests only read the committed ``*.pt`` files.
Nothing from the reference is copied: only its inputs/outputs (tensors) are stored.
"""
import importlib
import os
import sys

import torch

REF = "/root/reference/codes"
OUT = os.path.dirname(os.path.abspath(__file__))


def import_ref(task):
    """Import `utils` (sde_utils) and the task-local `models.modules` of one config dir."""
    for k in list(sys.modules):
        if k == "models" or k.startswith("models.") or k == "utils" or k.startswith("utils."):
            del sys.modules[k]
    os.chdir(os.path.join(REF, "config", task))
    sys.path[:] = [p for p in sys.path if "/root/reference" not in p]
    sys.path.insert(0, os.path.join(REF, "config", task))
    sys.path.insert(0, REF)
    utils = importlib.import_module("utils")
    mods = importlib.import_module("models.modules")
    return utils, mods


def sched_dict(sde):
    return dict(thetas=sde.thetas.clone(), sigmas=sde.sigmas.clone(), thetas_cumsum=sde.thetas_cumsum.clone(),
                sigma_bars=sde.sigma_bars.clone(), dt=torch.as_tensor(sde.dt).clone(), max_sigma=float(sde.max_sigma))


def main():
    torch.set_num_threads(4)
    gold = {}
    utils, mods = import_ref("deraining")

    # 1. schedule known answers -------------------------------------------------------
    sch = []
    for (ms, T, s, eps) in [(10, 100, "cosine", 0.005), (10, 50, "cosine", 0.005), (50, 200, "cosine", 0.005),
                            (30, 100, "linear", 0.005), (0.1, 20, "constant", 0.01), (10, 400, "cosine", 0.005)]:
        sde = utils.IRSDE(max_sigma=ms, T=T, schedule=s, eps=eps, device="cpu")
        sch.append(dict(args=(ms, T, s, eps), **sched_dict(sde)))
    gold["irsde_schedules"] = sch
    dsch = []
    for (ms, T, s) in [(75, 100, "cosine"), (50, 50, "linear"), (1, 30, "cosine")]:
        sde = utils.DenoisingSDE(max_sigma=ms, T=T, schedule=s, device="cpu")
        d = dict(args=(ms, T, s), **sched_dict(sde))
        d["optimal_t"] = {sg: int(sde.get_optimal_timestep(sg)) for sg in (15, 25, 50)} if ms == 75 else {}
        dsch.append(d)
    gold["dsde_schedules"] = dsch

    # 2. single sampler steps (teacher-forced) ----------------------------------------
    g = torch.Generator().manual_seed(7)
    sde = utils.IRSDE(max_sigma=10, T=100, schedule="cosine", eps=0.005, device="cpu")
    shp = (2, 3, 5, 7)
    x, mu, noise = [torch.randn(shp, generator=g) for _ in range(3)]
    sde.set_mu(mu)
    steps = []
    for t in (100, 50, 2, 1):
        torch.manual_seed(100 + t)
        z = torch.randn(shp)
        torch.manual_seed(100 + t)
        out_sde = sde.reverse_sde_step(x, sde.get_score_from_noise(noise, t), t)
        out_ode = sde.reverse_ode_step(x, sde.get_score_from_noise(noise, t), t)
        torch.manual_seed(100 + t)
        out_post = sde.reverse_posterior_step(x, noise, t)
        steps.append(dict(t=t, z=z, sde=out_sde, ode=out_ode, posterior=out_post))
    gold["irsde_steps"] = dict(x=x, mu=mu, noise=noise, steps=steps, args=(10, 100, "cosine", 0.005))

    dsde = utils.DenoisingSDE(max_sigma=75, T=100, schedule="cosine", device="cpu")
    dsteps = []
    for t in (100, 38, 2, 1):
        torch.manual_seed(200 + t)
        z = torch.randn(shp)
        torch.manual_seed(200 + t)
        score = dsde.get_score_from_noise(noise, t)
        o_sde = dsde.reverse_sde_step(x, score, t)
        o_ode = dsde.reverse_ode_step(x, score, t)
        dsteps.append(dict(t=t, z=z, sde=o_sde, ode=o_ode))
    gold["dsde_steps"] = dict(x=x, noise=noise, steps=dsteps, args=(75, 100, "cosine"))

    # 3. ConditionalUNet forward (deraining variant) ----------------------------------
    torch.manual_seed(0)
    net = mods.ConditionalUNet(3, 3, 8, depth=2).eval()
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    # make gains / biases non-trivial so index mistakes cannot hide
    gg = torch.Generator().manual_seed(3)
    for k in sd:
        if k.endswith(".g"):
            sd[k] = 1 + 0.2 * torch.randn(sd[k].shape, generator=gg)
        if k.endswith("bias"):
            sd[k] = sd[k] + 0.05 * torch.randn(sd[k].shape, generator=gg)
    net.load_state_dict(sd)
    xt = torch.rand(2, 3, 18, 27, generator=g)
    cond = torch.rand(2, 3, 18, 27, generator=g)
    with torch.no_grad():
        y_int = net(xt, cond, 37)
        y_vec = net(xt, cond, torch.tensor([5, 37]))
    gold["unet_cond"] = dict(nf=8, depth=2, state=sd, xt=xt, cond=cond, t_int=37, y_int=y_int,
                             t_vec=torch.tensor([5, 37]), y_vec=y_vec)

    # 4. full chains through the reference sampler + network --------------------------
    sde = utils.IRSDE(max_sigma=10, T=20, schedule="cosine", eps=0.005, device="cpu")
    sde.set_model(net)
    lq = torch.rand(1, 3, 16, 16, generator=g)
    sde.set_mu(lq)
    torch.manual_seed(11)
    xT = sde.noise_state(lq)
    chains = {}
    for mode in ("sde", "ode", "posterior"):
        torch.manual_seed(12)
        zs = torch.stack([torch.randn_like(xT) for _ in range(20)])
        torch.manual_seed(12)
        with torch.no_grad():
            x0 = getattr(sde, "reverse_" + mode)(xT)
        torch.manual_seed(12)
        with torch.no_grad():
            x5 = getattr(sde, "reverse_" + mode)(xT, T=5)
        chains[mode] = dict(x0=x0, x0_T5=x5, zs=zs)
    gold["irsde_chain"] = dict(args=(10, 20, "cosine", 0.005), lq=lq, xT=xT, chains=chains)

    # 5. denoising-sde variant (no cond, full Attention mid) --------------------------
    utils2, mods2 = import_ref("denoising-sde")
    torch.manual_seed(1)
    net2 = mods2.ConditionalUNet(3, 3, 8, depth=2).eval()
    sd2 = {k: v.clone() for k, v in net2.state_dict().items()}
    for k in sd2:
        if k.endswith(".g"):
            sd2[k] = 1 + 0.2 * torch.randn(sd2[k].shape, generator=gg)
        if k.endswith("bias"):
            sd2[k] = sd2[k] + 0.05 * torch.randn(sd2[k].shape, generator=gg)
    net2.load_state_dict(sd2)
    xd = torch.rand(2, 3, 14, 16, generator=g)
    with torch.no_grad():
        yd = net2(xd, 9)
    dsde = utils2.DenoisingSDE(max_sigma=75, T=30, schedule="cosine", device="cpu")
    dsde.set_model(net2)
    torch.manual_seed(21)
    zs = torch.stack([torch.randn_like(xd) for _ in range(30)])
    Tstar = int(dsde.get_optimal_timestep(25))
    torch.manual_seed(21)
    with torch.no_grad():
        xo_sde = dsde.reverse_sde(xd, T=Tstar)
        xo_ode = dsde.reverse_ode(xd, T=Tstar)
    gold["unet_dsde"] = dict(nf=8, depth=2, state=sd2, x=xd, t_int=9, y=yd, args=(75, 30, "cosine"), Tstar=Tstar,
                             zs=zs, x0_sde=xo_sde, x0_ode=xo_ode)

    sys.path.insert(0, os.path.dirname(OUT))
    import _golden
    _golden.save(gold, "reference_golden.pt")
    n = os.path.getsize(os.path.join(OUT, "reference_golden.pt"))
    print("wrote reference_golden.pt", n, "bytes")


if __name__ == "__main__":
    main()
