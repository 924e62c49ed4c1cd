"""Training-time use without a GPU: ``infer_nafnet_config`` on the reference's own NAFNets as every shipped Refusion config
builds them, and the launcher's ``train.py`` mode on the staged task trees (samplers swapped, the trained networks left as
the reference's classes, the frozen autoencoder native).  Skipped where oracle/_ref is not staged."""
import glob
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, "oracle", "_ref", "codes", "config")

# which staged tree holds the architecture a task's yml builds (deblurring ... sisr share the deraining class)
ARCH = {"denoising-sde": "denoising-sde", "latent-dehazing": "latent-dehazing"}
YMLS = sorted(glob.glob(os.path.join(CONFIG, t, "options", "*", "refusion.yml"))
              for t in ("deraining", "deblurring", "deshadow", "inpainting", "sisr", "denoising-sde"))
YMLS = [y for ys in YMLS for y in ys] + sorted(glob.glob(os.path.join(CONFIG, "latent-dehazing", "options", "*", "*", "nasde.yml")))


def _need_ref():
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", ".staged")):
        pytest.skip("oracle/_ref not staged")


def _infer_in_tree(task, settings, extra=""):
    """infer_nafnet_config of the reference ConditionalNAFNet of a task tree, built on the meta device (shapes only) from
    each setting, in a fresh interpreter that imports the tree's ``models.modules`` the way its scripts do."""
    import json
    tree = os.path.join(CONFIG, ARCH.get(task, "deraining"))
    code = ("import sys, os, json, torch; sys.path[:0] = [%r, %r, os.path.join(%r, '..', '..')]; import irsde_b200; "
            "from irsde_b200 import run; run._stub_missing(); os.chdir(%r); import models.modules as M; out = []\n"
            "for s in json.loads(sys.argv[1]):\n"
            "    with torch.device('meta'): sd = M.ConditionalNAFNet(**s).state_dict()\n"
            "    %s\n"
            "    out.append(irsde_b200.infer_nafnet_config(sd))\n"
            "print('RESULT' + json.dumps(out))" % (ROOT, tree, tree, tree, extra or "pass"))
    p = subprocess.run([sys.executable, "-c", code, json.dumps(settings)], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]
    res = json.loads(p.stdout.split("RESULT", 1)[1])
    return [tuple(r) if r is not None else None for r in res]


def _yml_cases():
    _need_ref()
    import yaml
    out = []
    for y in YMLS:
        task = os.path.relpath(y, CONFIG).split(os.sep)[0]
        setting = yaml.safe_load(open(y))["network_G"]["setting"]
        out.append((os.path.relpath(y, CONFIG), task, setting))
    assert len(out) == 14, [o[0] for o in out]     # train + test refusion.yml of six tasks, train + test nasde.yml
    return out


def test_infer_nafnet_config_reads_every_shipped_refusion_network():
    cases = _yml_cases()
    for task in sorted({c[1] for c in cases}):
        mine = [c for c in cases if c[1] == task]
        got = _infer_in_tree(task, [c[2] for c in mine])
        for (name, _, setting), g in zip(mine, got):
            want = (setting.get("img_channel", 3), setting["width"], setting.get("middle_blk_num", 1),
                    list(setting["enc_blk_nums"]), list(setting["dec_blk_nums"]),
                    "denoising" if task == "denoising-sde" else "conditional")
            assert g == want, (name, g, want)


def test_infer_nafnet_config_declines_other_state_dicts():
    import irsde_b200
    _need_ref()
    setting = dict(width=16, enc_blk_nums=[1, 1], middle_blk_num=1, dec_blk_nums=[1, 1])
    unet = irsde_b200.ConditionalUNet(3, 3, 8, depth=2).state_dict()
    assert irsde_b200.infer_unet_config(unet) is not None and irsde_b200.infer_nafnet_config(unet) is None
    # stereo-sr puts a cross-view fusion module (SCAM) after the blocks, latent-bokeh a lens MLP beside the time MLP; the
    # same keys in another order are not the reference's layout either
    extras = {
        "plain": "pass",
        "fusion": "sd['fusion.0.l_proj1.weight'] = torch.zeros(16, 16, 1, 1, device='meta')",
        "cam_mlp": "sd = type(sd)([(k, v) for k, v in sd.items()][:4] + [('cam_mlp.0.weight', torch.zeros(64, 2))] + "
                   "[(k, v) for k, v in sd.items()][4:])",
        "reordered": "sd = type(sd)(sorted(sd.items()))",
    }
    for label, extra in extras.items():
        (got,) = _infer_in_tree("deraining", [setting], extra)
        assert (got is not None) == (label == "plain"), (label, got)


def _install(task, check):
    code = ("import sys, os; sys.path.insert(0, %r); import irsde_b200; from irsde_b200 import run; os.chdir(%r); "
            "u, m = run.install(os.getcwd(), train=True); from models import networks; import timm; " % (ROOT, os.path.join(CONFIG, task))
            + check + "; print('ok')")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr[-3000:]


@pytest.mark.parametrize("task", ["deraining", "denoising-sde", "latent-dehazing"])
def test_launcher_train_mode_keeps_the_reference_networks(task):
    """train.py through the launcher: our samplers, the reference's trainable network classes, timm importable."""
    _need_ref()
    check = ("assert u.IRSDE is irsde_b200.IRSDE and u.DenoisingSDE is irsde_b200.DenoisingSDE; "
             "assert m.ConditionalUNet.__module__ == 'models.modules.DenoisingUNet_arch'; "
             "assert m.ConditionalNAFNet.__module__ == 'models.modules.DenoisingNAFNet_arch'; "
             "net = networks.define_G({'network_G': {%r: 'ConditionalNAFNet', 'setting': dict(width=8, enc_blk_nums=[1], "
             "middle_blk_num=1, dec_blk_nums=[1])}}); assert not isinstance(net, irsde_b200.ConditionalUNet)"
             % ("which_model" if task == "latent-dehazing" else "which_model_G"))
    _install(task, check)


def test_launcher_train_mode_builds_the_frozen_autoencoder_natively():
    """latent-dehazing's define_L returns irsde_b200.UNet, initialised from the reference's own module so the global
    generator ends where the reference's construction leaves it; define_G still builds the reference's classes."""
    _need_ref()
    check = ("import torch, yaml; opt = yaml.safe_load(open('options/dehazing/train/nasde.yml')); "
             "assert m.UNet.__module__ == 'models.modules.UNet_arch'; "
             "torch.manual_seed(3); ref = m.UNet(**opt['network_L']['setting']); after_ref = torch.rand(4); "
             "torch.manual_seed(3); L = networks.define_L(opt); after_ours = torch.rand(4); "
             "assert isinstance(L, irsde_b200.UNet) and torch.equal(after_ref, after_ours); "
             "assert all(torch.equal(a, b) for a, b in zip(L.state_dict().values(), ref.state_dict().values())); "
             "assert list(L.state_dict()) == list(ref.state_dict()); "
             "g = networks.define_G({'network_G': {'which_model': 'UNet', 'setting': opt['network_L']['setting']}}); "
             "assert not isinstance(g, irsde_b200.UNet)")
    _install("latent-dehazing", check)


def test_timm_stand_in_refuses_to_build_a_dit():
    _need_ref()
    _install("latent-dehazing", "import pytest; M = __import__('models.modules', fromlist=['x']); "
                                "pytest.raises(ImportError, M.DiT_S_8, input_size=32)")
