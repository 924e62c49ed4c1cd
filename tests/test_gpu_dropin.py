"""Drop-in proof (SURVEY 8 b): the reference's own `codes/config/deraining/test.py` (test.py:67-72,93-110), UNMODIFIED,
run twice on three synthetic PNG pairs with a random-weight checkpoint -
  (A) through `python -m irsde_b200.run` (IRSDE + ConditionalUNet swapped for the native sm_90a sampler, fp32 parity mode),
  (B) through `python -m irsde_b200.run --reference` (nothing swapped: the reference on PyTorch eager, same GPU) -
with the same seed.  The PNGs both runs write must agree to within one grey level (uint8 rounding of a <=1e-3 difference).
Needs the reference staged under oracle/_ref (oracle/make_ref.py, done by __graft_entry__.build()); skipped without it."""
import os
import shutil
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")

YML = """name: dropin
suffix: ~
model: denoising
distortion: derain
gpu_ids: [0]
sde:
  max_sigma: 10
  T: 12
  schedule: cosine
  eps: 0.005
  sampling_mode: {mode}
degradation:
  sigma: 25
  noise_type: G
  scale: 4
datasets:
  test1:
    name: Val_Dataset
    mode: LQGT
    dataroot_GT: {root}/data/GT
    dataroot_LQ: {root}/data/LQ
network_G:
  which_model_G: ConditionalUNet
  setting:
    in_nc: 3
    out_nc: 3
    nf: 16
    depth: 2
path:
  pretrain_model_G: {root}/ckpt.pth
"""


def _run(tree, launcher_args, env_extra, log):
    env = dict(os.environ)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    env.update(env_extra)
    cwd = os.path.join(tree, "codes", "config", "deraining")
    cmd = [sys.executable, "-m", "irsde_b200.run"] + launcher_args + ["test.py", "-opt=" + os.path.join(tree, "opt.yml")]
    p = subprocess.run(cmd, cwd=cwd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    open(log, "w").write(p.stdout)
    assert p.returncode == 0, p.stdout[-3000:]
    return p.stdout


@pytest.mark.parametrize("mode", ["posterior", "sde"])
def test_reference_test_py_runs_unchanged(tmp_path, mode):
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
        os.makedirs(os.path.join(tree, "data", "LQ"))
        rng = np.random.RandomState(0)
        for i, (h, w) in enumerate([(64, 64), (48, 80), (50, 38)]):   # the last two are not multiples of 4: reflect pad
            gt = (rng.rand(h, w, 3) * 255).astype(np.uint8)
            lq = np.clip(gt.astype(np.int32) + rng.randint(-30, 30, gt.shape), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(tree, "data", "GT", "img%d.png" % i), gt)
            cv2.imwrite(os.path.join(tree, "data", "LQ", "img%d.png" % i), lq)
        open(os.path.join(tree, "opt.yml"), "w").write(YML.format(root=tree, mode=mode))
        trees[arm] = tree
    # checkpoint: the REFERENCE network's own state dict (default init, seed 0), saved the way save_network does
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    code = ("import sys, torch; sys.path.insert(0, %r); import ref_loader; u, m = ref_loader.load('deraining'); torch.manual_seed(0); "
            "net = m.ConditionalUNet(3, 3, 16, 2); torch.save({k: v.cpu() for k, v in net.state_dict().items()}, sys.argv[1])"
            % os.path.join(ROOT, "oracle"))
    for tree in trees.values():
        subprocess.run([sys.executable, "-c", code, os.path.join(tree, "ckpt.pth")], check=True, timeout=300)
    out_native = _run(trees["native"], ["--seed", "123"], {"IRSDE_B200_PRECISION": "fp32"}, str(tmp_path / "native.log"))
    out_ref = _run(trees["reference"], ["--seed", "123", "--reference"], {"NVIDIA_TF32_OVERRIDE": "0"}, str(tmp_path / "ref.log"))
    assert "irsde_b200" not in out_ref
    res = {}
    for arm, tree in trees.items():
        d = os.path.join(tree, "results", "deraining", "dropin", "Val_Dataset")
        assert os.path.isdir(d), os.listdir(os.path.join(tree))
        res[arm] = {f: cv2.imread(os.path.join(d, f), cv2.IMREAD_UNCHANGED) for f in sorted(os.listdir(d)) if f.endswith(".png")}
    assert sorted(res["native"]) == sorted(res["reference"]) and len(res["native"]) == 9   # output + _LQ + _HQ per image
    worst = 0
    for f in res["native"]:
        a, b = res["native"][f].astype(np.int32), res["reference"][f].astype(np.int32)
        assert a.shape == b.shape
        worst = max(worst, int(np.abs(a - b).max()))
        if f.endswith("_LQ.png") or f.endswith("_HQ.png"):
            assert np.array_equal(a, b)
    assert worst <= 1, "restored images differ by %d grey levels" % worst
    # both logs report the same metrics line format (the script ran to its end in both arms)
    assert "Average PSNR/SSIM" in out_native and "Average PSNR/SSIM" in out_ref


def test_validation_sampling_adopts_reference_module_during_training():
    """SURVEY 8 f-4 (train.py:214-215,236,261-281): the reference's PyTorch ConditionalUNet keeps being trained by autograd;
    `sde.set_model(DataParallel(net))` + `model.eval()` + `sde.reverse_posterior(...)` must sample through the native
    kernels with the module's CURRENT weights (before and after an optimizer step), and `generate_random_states` must give
    the reference's states bit for bit."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    if not os.path.exists(os.path.join(REF, ".staged")):
        pytest.skip("oracle/_ref not staged")
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    sys.path.insert(0, ROOT)
    import ref_loader
    rutil, rmods = ref_loader.load("deraining")
    import irsde_b200
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    ref_net = rmods.ConditionalUNet(3, 3, 16, 2).to(dev)
    wrapped = torch.nn.DataParallel(ref_net, device_ids=[0])
    ours = irsde_b200.IRSDE(10, 12, schedule="cosine", eps=0.005, device=dev)
    theirs = rutil.IRSDE(max_sigma=10, T=12, schedule="cosine", eps=0.005, device=dev)
    ours.set_model(wrapped)
    theirs.set_model(wrapped)
    g = torch.Generator().manual_seed(1)
    GT, LQ = torch.rand(2, 3, 24, 40, generator=g), torch.rand(2, 3, 24, 40, generator=g)

    # ---- train.py:236  generate_random_states: same generator calls, bit-identical states
    torch.manual_seed(5)
    t_ref, s_ref = theirs.generate_random_states(x0=GT, mu=LQ)
    torch.manual_seed(5)
    t_our, s_our = ours.generate_random_states(x0=GT, mu=LQ)
    assert torch.equal(t_ref, t_our) and torch.equal(s_ref, s_our)

    opt = torch.optim.SGD(ref_net.parameters(), lr=1e-2)

    def validate():
        wrapped.eval()
        outs = []
        for sde in (theirs, ours):
            sde.set_mu(LQ.to(dev))
            torch.manual_seed(9)
            with torch.no_grad():
                outs.append(sde.reverse_posterior(LQ.to(dev) + 0.03))
        wrapped.train()
        return outs

    a_ref, a_our = validate()
    assert (a_ref - a_our).abs().max().item() < 1e-3
    shadow = getattr(ref_net, "_irsde_b200_shadow", None)
    assert shadow is not None and shadow is not False and shadow.launch_count() > 0     # the native kernels ran
    # ---- one real training step through the reference's autograd forward (train.py:239 optimize_parameters)
    ref_net.train()
    ts, states = theirs.generate_random_states(x0=GT, mu=LQ)
    noise = theirs.noise_fn(states, ts.squeeze().to(dev))
    loss = noise.pow(2).mean()
    loss.backward()
    opt.step()
    b_ref, b_our = validate()
    assert (b_ref - b_our).abs().max().item() < 1e-3           # the shadow picked up the updated weights
    assert (b_ref - a_ref).abs().max().item() > 1e-4           # and the step did change the result
