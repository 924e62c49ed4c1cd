"""The denoising-sde task's ConditionalNAFNet (DenoisingNAFNet here) on the host: the oracle against the reference's own
outputs, the state-dict contract, and the launcher's choice of class per task directory."""
import os
import subprocess
import sys

import pytest
import torch

from oracle import irsde_oracle as O
import _nafnet_denoising_oracle as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "reference_golden_nafnet_dsde.pt"), weights_only=True)


def _close(a, b, tol):
    d = (a - b).abs().max().item()
    assert d <= tol, d


def test_oracle_forward_and_chains_match_reference():
    g = _gold()
    c = g["cfg"]
    args = (c["width"], c["enc_blk_nums"], c["middle_blk_num"], c["dec_blk_nums"])
    _close(D.forward(g["state"], g["x"], g["t_int"], *args), g["y"], 1e-5)
    _close(D.forward(g["state"], g["x"], g["t_vec"], *args), g["y_vec"], 1e-5)
    shapes = D.param_shapes(c["img_channel"], c["width"], c["middle_blk_num"], c["enc_blk_nums"], c["dec_blk_nums"])
    assert list(shapes) == list(g["state"])
    assert all(tuple(g["state"][k].shape) == tuple(v) for k, v in shapes.items())
    sc = O.Schedule(*g["args"], kind="dsde")
    assert O.get_optimal_timestep(sc, g["sigma"]) == g["Tstar"] == 22
    net = lambda x, t: D.forward(g["state"], x, t, *args)
    _close(O.reverse_chain(sc, net, g["xn"], None, g["zs"], "dsde_sde", T=g["Tstar"]), g["x0_sde"], 2e-4)
    _close(O.reverse_chain(sc, net, g["xn"], None, g["zs"], "dsde_ode", T=g["Tstar"]), g["x0_ode"], 2e-4)


def test_denoising_nafnet_state_dict_contract():
    import irsde_b200
    g = _gold()
    net = irsde_b200.DenoisingNAFNet(**g["cfg"])
    assert isinstance(net, irsde_b200.ConditionalNAFNet) and net.variant == "denoising"
    sd = net.state_dict()
    assert list(sd.keys()) == list(g["state"].keys())
    assert all(tuple(sd[k].shape) == tuple(v.shape) for k, v in g["state"].items())
    net.load_state_dict(g["state"], strict=True)
    c = g["cfg"]
    assert irsde_b200.nafnet_param_shapes(c["img_channel"], c["width"], c["middle_blk_num"], c["enc_blk_nums"],
                                          c["dec_blk_nums"], "denoising")["intro.weight"] == (8, 3, 3, 3)
    # the conditional class keeps its layout and rejects this checkpoint
    with pytest.raises(RuntimeError):
        irsde_b200.ConditionalNAFNet(**c).load_state_dict(g["state"], strict=True)


def test_denoising_nafnet_needs_cuda():
    import irsde_b200
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    net = irsde_b200.DenoisingNAFNet(**_gold()["cfg"])
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 8, 8), 1)


@pytest.mark.parametrize("task,cls", [("denoising-sde", "DenoisingNAFNet"), ("deraining", "ConditionalNAFNet")])
def test_launcher_picks_nafnet_variant_per_task(task, cls):
    ref = os.path.join(ROOT, "oracle", "_ref", "codes", "config", task)
    if not os.path.isdir(ref):
        pytest.skip("oracle/_ref not staged")
    code = (
        "import sys, os; sys.path.insert(0, %r); import irsde_b200; from irsde_b200 import run; os.chdir(%r); "
        "u, m = run.install(%r); from models import networks; "
        "naf = networks.define_G({'network_G': {'which_model_G': 'ConditionalNAFNet', 'setting': dict(width=8, "
        "enc_blk_nums=[1], middle_blk_num=1, dec_blk_nums=[1])}}); "
        "assert type(naf) is irsde_b200.%s, type(naf); "
        "assert tuple(naf.state_dict()['intro.weight'].shape) == (8, %d, 3, 3); print('ok')"
        % (ROOT, ref, ref, cls, 3 if cls == "DenoisingNAFNet" else 6))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr[-2000:]
