"""Golden fixture for the denoising-sde task's ConditionalNAFNet (no condition input, intro over img_channel channels)
driven by DenoisingSDE, generated from the imported reference.
    python tests/golden/make_golden_nafnet_dsde.py
"""
import importlib.util
import os
import sys

import torch

OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, OUT)
from make_golden_nafnet import REF, load_arch  # noqa: E402


def load_sde_utils():
    """codes/utils/sde_utils.py by file path (the package __init__ pulls in every image helper)."""
    spec = importlib.util.spec_from_file_location("ref_sde_utils", os.path.join(REF, "utils", "sde_utils.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def main():
    torch.set_num_threads(4)
    arch = load_arch("denoising-sde")
    sde_utils = load_sde_utils()
    g = torch.Generator().manual_seed(7)
    cfg = dict(img_channel=3, width=8, middle_blk_num=1, enc_blk_nums=[1, 2], dec_blk_nums=[1, 1])
    torch.manual_seed(3)
    net = arch.ConditionalNAFNet(**cfg).eval()
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    for k in sd:  # beta/gamma are zero-initialised in the reference: make every branch matter
        if k.endswith("beta") or k.endswith("gamma"):
            sd[k] = 0.5 * torch.randn(sd[k].shape, generator=g)
        if k.endswith(".g"):
            sd[k] = 1 + 0.2 * torch.randn(sd[k].shape, generator=g)
    net.load_state_dict(sd)
    x = torch.rand(2, 3, 18, 23, generator=g)     # zero-padded to 20 x 24 inside the network
    t_vec = torch.tensor([3, 40])
    with torch.no_grad():
        y = net(x, 13)
        yv = net(x, t_vec)
    sde = sde_utils.DenoisingSDE(max_sigma=70, T=100, device="cpu")
    sde.set_model(net)
    Tstar = int(sde.get_optimal_timestep(25))
    xn = x + torch.randn(x.shape, generator=g) * (25 / 255)
    torch.manual_seed(21)
    zs = torch.stack([torch.randn_like(xn) for _ in range(Tstar)])   # the draws reverse_sde makes, in loop order
    torch.manual_seed(21)
    with torch.no_grad():
        x0_sde = sde.reverse_sde(xn, T=Tstar)
        x0_ode = sde.reverse_ode(xn, T=Tstar)
    gold = dict(cfg=cfg, state=sd, x=x, t_int=13, y=y, t_vec=t_vec, y_vec=yv, args=(70, 100), sigma=25, Tstar=Tstar,
                xn=xn, zs=zs, x0_sde=x0_sde, x0_ode=x0_ode)
    path = os.path.join(OUT, "reference_golden_nafnet_dsde.pt")
    torch.save(gold, path)
    print("wrote", os.path.getsize(path), "bytes; T* =", Tstar)


if __name__ == "__main__":
    main()
