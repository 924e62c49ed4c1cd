"""Drop-in proof for the denoising-sde task: the reference's own `codes/config/denoising-sde/test.py`, UNMODIFIED, run with
each of its two networks (options/test/ir-sde.yml: the denoising ConditionalUNet; options/test/refusion.yml: the denoising
ConditionalNAFNet) on three synthetic PNGs with a random-weight checkpoint -
  (A) through `python -m irsde_b200.run` (DenoisingSDE and the network swapped for the native sm_90a sampler, fp32),
  (B) through `python -m irsde_b200.run --reference` (nothing swapped: the reference on PyTorch eager, same GPU) -
with the same seed.  test.py always passes save_states=True, so both arms also leave the last image's ODE states behind.
Needs the reference staged under oracle/_ref (oracle/make_ref.py, done by __graft_entry__.build()); skipped without it."""
import os
import shutil
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")

# T >= 100: test.py passes save_states=True and the reference's state interval is T // 100
YML = """name: dropin
suffix: ~
model: denoising
gpu_ids: [0]
sde:
  max_sigma: 70
  T: 100
degradation:
  sigma: 15
  noise_type: G
datasets:
  test1:
    name: Val
    mode: GT
    dataroot_GT: {root}/data/GT
network_G:
{net}
path:
  pretrain_model_G: {root}/ckpt.pth
"""
NETS = {
    "unet": ("  which_model_G: ConditionalUNet\n  setting:\n    in_nc: 3\n    out_nc: 3\n    nf: 16\n    depth: 2",
             "net = m.ConditionalUNet(3, 3, 16, 2)"),
    "nafnet": ("  which_model_G: ConditionalNAFNet\n  setting:\n    width: 16\n    enc_blk_nums: [1, 1]\n    middle_blk_num: 1\n"
               "    dec_blk_nums: [1, 1]",
               "net = m.ConditionalNAFNet(width=16, enc_blk_nums=[1, 1], middle_blk_num=1, dec_blk_nums=[1, 1])"),
}
# beta / gamma are zero-initialised in the reference (every NAFBlock would be the identity): give them values
CKPT = ("import sys, torch; sys.path.insert(0, %r); import ref_loader; u, m = ref_loader.load('denoising-sde'); "
        "torch.manual_seed(0); %s; sd = {k: v.cpu() for k, v in net.state_dict().items()}; g = torch.Generator().manual_seed(1); "
        "sd.update({k: 0.3 * torch.randn(v.shape, generator=g) for k, v in sd.items() if k.endswith(('beta', 'gamma'))}); "
        "torch.save(sd, sys.argv[1])")


def _run(tree, launcher_args, env_extra, log):
    env = dict(os.environ)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    env.update(env_extra)
    cwd = os.path.join(tree, "codes", "config", "denoising-sde")
    cmd = [sys.executable, "-m", "irsde_b200.run"] + launcher_args + ["test.py", "-opt=" + os.path.join(tree, "opt.yml")]
    p = subprocess.run(cmd, cwd=cwd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    open(log, "w").write(p.stdout)
    assert p.returncode == 0, p.stdout[-3000:]
    return p.stdout


def _read_dir(d, ext):
    import cv2
    assert os.path.isdir(d), d
    return {f: cv2.imread(os.path.join(d, f), cv2.IMREAD_UNCHANGED) for f in sorted(os.listdir(d)) if f.endswith(ext)}


@pytest.mark.parametrize("net", ["unet", "nafnet"])
def test_denoising_sde_test_py_runs_unchanged(tmp_path, net):
    import cv2
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    if not os.path.exists(os.path.join(REF, ".staged")):
        pytest.skip("oracle/_ref not staged (python oracle/make_ref.py next to the reference checkout)")
    trees = {}
    for arm in ("native", "reference"):
        tree = str(tmp_path / arm)
        shutil.copytree(REF, tree)
        os.makedirs(os.path.join(tree, "data", "GT"))
        rng = np.random.RandomState(0)
        for i, (h, w) in enumerate([(64, 64), (48, 82), (50, 38)]):   # the last two are not multiples of 4: padded
            cv2.imwrite(os.path.join(tree, "data", "GT", "img%d.png" % i), (rng.rand(h, w, 3) * 255).astype(np.uint8))
        open(os.path.join(tree, "opt.yml"), "w").write(YML.format(root=tree, net=NETS[net][0]))
        subprocess.run([sys.executable, "-c", CKPT % (os.path.join(ROOT, "oracle"), NETS[net][1]), os.path.join(tree, "ckpt.pth")],
                       check=True, timeout=300)
        trees[arm] = tree
    out_native = _run(trees["native"], ["--seed", "123"], {"IRSDE_B200_PRECISION": "fp32"}, str(tmp_path / "native.log"))
    out_ref = _run(trees["reference"], ["--seed", "123", "--reference"], {"NVIDIA_TF32_OVERRIDE": "0"}, str(tmp_path / "ref.log"))
    assert "irsde_b200" not in out_ref
    worst = 0
    for sub, ext, n in ((os.path.join("results", "denoising-sde", "dropin", "Val_sigma15"), ".png", 6),
                        (os.path.join("results", "denoising-sde", "dropin", "Val_sigma15"), ".tif", 3),
                        (os.path.join("codes", "config", "denoising-sde", "ode_state"), ".png", None)):
        res = {arm: _read_dir(os.path.join(tree, sub), ext) for arm, tree in trees.items()}
        assert sorted(res["native"]) == sorted(res["reference"]) and res["native"], (sub, ext)
        assert n is None or len(res["native"]) == n, sorted(res["native"])
        for f in res["native"]:
            a, b = res["native"][f].astype(np.int32), res["reference"][f].astype(np.int32)
            assert a.shape == b.shape, f
            if f.endswith(("_noisy.png", "_clean.png")):
                assert np.array_equal(a, b), f
            else:
                worst = max(worst, int(np.abs(a - b).max()))
    assert worst <= 1, "restored images / ODE states differ by %d grey levels" % worst
    assert "Average PSNR/SSIM" in out_native and "Average PSNR/SSIM" in out_ref
