"""Training-time drop-in (train.py:214-215,238-241,261-281): the reference's PyTorch networks keep being trained by autograd
while validation samples them on the native kernels through an adopted shadow.

1. Adoption of each NAFNet form, in fp32 on the pattern of test_gpu_dropin.py's UNet test: the reference module wrapped in
   DataParallel, one validation pass through the reference sampler and ours, one real Lion step (the optimizer the
   refusion / nasde ymls select) through the reference's autograd forward, a second pass.
2. The reference's unmodified train.py, run through ``python -m irsde_b200.run --seed S`` (in-process, so the shadows can be
   inspected afterwards) and through ``--reference``, on a copy of oracle/_ref each, with a generated yml and dataset.

Needs the reference staged under oracle/_ref (oracle/make_ref.py, done by __graft_entry__.build()); skipped without it."""
import json
import math
import os
import shutil
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
SMALL_NAF = dict(width=16, enc_blk_nums=[1, 1, 1, 2], middle_blk_num=1, dec_blk_nums=[1, 1, 1, 1])


def _need_gpu_and_ref():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    if not os.path.exists(os.path.join(REF, ".staged")):
        pytest.skip("oracle/_ref not staged")


def _card():
    import torch
    p = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return "%s, power limit %s" % (torch.cuda.get_device_name(0), p.stdout.strip() or "unknown")


def _load_task(task):
    """(utils, models.modules, models.optimizer) of a staged task tree; the previous task's ``models`` package is dropped
    first (every task tree has its own under the same name)."""
    import importlib
    for name in [n for n in sys.modules if n == "models" or n.startswith("models.")]:
        del sys.modules[name]
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import ref_loader
    from irsde_b200 import run
    run._stub_missing()      # latent-dehazing's models.modules imports timm (DiT_arch)
    utils, mods = ref_loader.load(task)
    return utils, mods, importlib.import_module("models.optimizer")


FORMS = ["deraining", "denoising-sde", "latent-dehazing"]


@pytest.fixture
def task_modules():
    """Put back the ``models`` package and sys.path the test found: other tests load their own task tree by name."""
    def mine():
        return {n: m for n, m in sys.modules.items() if n == "models" or n.startswith("models.")}
    saved, path = mine(), list(sys.path)
    yield
    for n in mine():
        del sys.modules[n]
    sys.modules.update(saved)
    sys.path[:] = path


@pytest.mark.parametrize("task", FORMS)
def test_nafnet_adoption_through_training(task, task_modules):
    _need_gpu_and_ref()
    import torch
    import irsde_b200
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        _adoption_case(task, torch, irsde_b200)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


def _adoption_case(task, torch, irsde_b200):
    rutil, rmods, ropt = _load_task(task)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(1)
    torch.manual_seed(0)
    if task == "denoising-sde":
        ref_net = rmods.ConditionalNAFNet(**SMALL_NAF).to(dev)
        theirs, ours = rutil.DenoisingSDE(max_sigma=50, T=12, schedule="cosine", device=dev), \
            irsde_b200.DenoisingSDE(50, 12, schedule="cosine", device=dev)
        images = [torch.rand(1, 3, 48, 64, generator=g) for _ in range(2)]
        xs = [(im + torch.randn(im.shape, generator=g) * 50 / 255).to(dev) for im in images]

        def chain(sde, i):
            return sde.reverse_ode(xs[i])

        def train_noise(x, t):
            return wrapped(x, t)
    elif task == "deraining":
        ref_net = rmods.ConditionalNAFNet(**SMALL_NAF).to(dev)
        theirs, ours = rutil.IRSDE(max_sigma=50, T=12, schedule="cosine", eps=0.005, device=dev), \
            irsde_b200.IRSDE(50, 12, schedule="cosine", eps=0.005, device=dev)
        mus = [torch.rand(1, 3, 48, 64, generator=g).to(dev) for _ in range(2)]
        xs = [mu + torch.randn(mu.shape, generator=g).to(dev) * 50 / 255 for mu in mus]

        def chain(sde, i):      # model.test(sde) default: posterior sampling
            sde.set_mu(mus[i])
            return sde.reverse_posterior(xs[i])

        def train_noise(x, t):
            return theirs.noise_fn(x, t)
    else:   # the latent NAFNet over the staged pretrained autoencoder's latents
        ae = rmods.UNet(in_ch=3, out_ch=3, ch=8, ch_mult=[4, 8, 8, 16], embed_dim=8)
        ae.load_state_dict(torch.load(os.path.join(REF, "codes", "config", task, "pretrained_models", "latent-dehazing.pth")))
        ae = ae.to(dev).eval()
        torch.manual_seed(0)
        ref_net = rmods.ConditionalNAFNet(img_channel=8, **SMALL_NAF).to(dev)
        theirs, ours = rutil.IRSDE(max_sigma=50, T=12, schedule="cosine", eps=0.005, device=dev), \
            irsde_b200.IRSDE(50, 12, schedule="cosine", eps=0.005, device=dev)
        with torch.no_grad():
            enc = [ae.encode(torch.rand(1, 3, 128, 128, generator=g).to(dev)) for _ in range(2)]
        mus = [z for z, _ in enc]
        xs = [mu + torch.randn(mu.shape, generator=g).to(dev) * 50 / 255 for mu in mus]

        def chain(sde, i):      # the sampled latent, and the image the autoencoder decodes from it
            sde.set_mu(mus[i])
            z = sde.reverse_sde(xs[i])
            return z, ae.decode(z, enc[i][1])

        def train_noise(x, t):
            return theirs.noise_fn(x, t)
    wrapped = torch.nn.DataParallel(ref_net, device_ids=[0])
    theirs.set_model(wrapped)
    ours.set_model(wrapped)

    def validate(first):
        wrapped.eval()
        outs, states = [], []
        for sde in (theirs, ours):
            torch.manual_seed(9)
            torch.cuda.manual_seed(9)
            with torch.no_grad():
                outs.append([chain(sde, i) for i in range(len(xs))])
            states.append((torch.get_rng_state(), torch.cuda.get_rng_state(0)))
        wrapped.train()
        if first:   # adoption (with its probe) happened inside our arm: the global generators are where the reference left them
            assert torch.equal(states[0][0], states[1][0]) and torch.equal(states[0][1], states[1][1])
        return outs

    def agree(refs, ours):
        for r, o in zip(refs, ours):
            if isinstance(r, tuple):    # latent: the decoder amplifies a latent far from the data (outputs ~1e3 here)
                (r, rd), (o, od) = r, o
                assert ((rd - od).abs().max() / rd.abs().max()).item() < 1e-4
            assert (r - o).abs().max().item() < 1e-3

    a_ref, a_our = validate(True)
    agree(a_ref, a_our)
    shadow = getattr(ref_net, "_irsde_b200_shadow", None)
    assert isinstance(shadow, irsde_b200.ConditionalNAFNet) and shadow.launch_count() > 0     # the native kernels ran
    assert shadow.upload_count() == 1                       # the second image of the pass did not re-upload
    assert isinstance(shadow, irsde_b200.DenoisingNAFNet) == (task == "denoising-sde")
    assert shadow.latent == (task == "latent-dehazing")
    chosen = "latent" if shadow.latent else "plain"
    margins = {k: e / shadow.probe_bound for k, e in shadow.probe_errors.items() if k != chosen}
    print("%s: probe error of the chosen form %.2e (bound %.0e); wrong forms' error / bound: %s"
          % (task, shadow.probe_errors[chosen], shadow.probe_bound, {k: round(v, 1) for k, v in margins.items()}))
    assert all(m > 1 for m in margins.values())
    # the probe left the module as validate() drives it (train() restored after the pass) and its parameters in place
    assert all(m.training for m in ref_net.modules()) and all(p.numel() > 0 for p in ref_net.parameters())

    # one real training step through the reference's autograd forward (optimize_parameters), with the refusion ymls' Lion
    opt = ropt.Lion(ref_net.parameters(), lr=1e-3, weight_decay=0.01, betas=(0.9, 0.99))
    wrapped.train()
    x0 = torch.cat(xs[:1]).detach()
    ts = torch.tensor([7], device=dev)
    if task != "denoising-sde":
        theirs.set_mu(mus[0])
    loss = train_noise(x0, ts).pow(2).mean()
    loss.backward()
    opt.step()
    b_ref, b_our = validate(False)
    agree(b_ref, b_our)                                     # the shadow picked up the updated weights
    first = (lambda v: v[0] if isinstance(v, tuple) else v)
    assert max((first(b) - first(a)).abs().max().item() for a, b in zip(a_ref, b_ref)) > 1e-4   # and the step changed them
    assert shadow.upload_count() == 2                       # once per validation pass
    assert ref_net._irsde_b200_shadow is shadow


# ---------------------------------------------------------------------------------------------------------------------------
# 2. The unmodified train.py through the launcher

DRIVER = r'''
import json, os, sys, time
root, out_json, argv = sys.argv[1], sys.argv[2], sys.argv[3:]
sys.path.insert(0, root)
import torch
from irsde_b200 import run, shadow
script_dir = os.path.dirname(os.path.abspath([a for a in argv if not a.startswith("--") and a.endswith(".py")][0]))
for p in (script_dir, os.path.abspath(os.path.join(script_dir, "..", ".."))):
    sys.path.insert(0, p)
run._stub_missing()
import data

passes = []


class TimedLoader:
    """The validation loader, timing each full pass over it (train.py:264-279: sampling, decode, PSNR)."""

    def __init__(self, dl):
        self.dl = dl

    def __len__(self):
        return len(self.dl)

    def __iter__(self):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        for b in self.dl:
            yield b
        torch.cuda.synchronize()
        free, total = torch.cuda.mem_get_info()
        passes.append(dict(seconds=time.perf_counter() - t0, torch_peak_bytes=torch.cuda.max_memory_allocated(),
                           device_used_bytes=total - free))


create_dataloader = data.create_dataloader
data.create_dataloader = lambda ds, o, opt=None, sampler=None: (
    TimedLoader(create_dataloader(ds, o, opt, sampler)) if o["phase"] == "val" else create_dataloader(ds, o, opt, sampler))
shadows = []
adopt = shadow.adopt


def recording_adopt(module, precision=None):
    sh = adopt(module, precision)
    shadows.append(sh)
    return sh


shadow.adopt = recording_adopt
run.main(argv)
json.dump(dict(passes=passes, shadows=[None if s is None else dict(
    cls=type(s).__name__, latent=bool(getattr(s, "latent", False)), launches=s.launch_count(), uploads=s.upload_count(),
    probe_errors=getattr(s, "probe_errors", None)) for s in shadows]), open(out_json, "w"))
'''

CASES = {
    "deraining-refusion": dict(task="deraining", yml="options/train/refusion.yml", size=64, net=SMALL_NAF),
    "deraining-ir-sde": dict(task="deraining", yml="options/train/ir-sde.yml", size=64, net=dict(in_nc=3, out_nc=3, nf=16, depth=2)),
    "denoising-sde-refusion": dict(task="denoising-sde", yml="options/train/refusion.yml", size=64, net=SMALL_NAF),
    "latent-dehazing-nasde": dict(task="latent-dehazing", yml="options/dehazing/train/nasde.yml", size=128,
                                  net=dict(SMALL_NAF, img_channel=8)),
}
NITER, VAL_FREQ = 4, 2


def _write_tree(tree, case):
    import cv2
    import numpy as np
    import yaml
    shutil.copytree(REF, tree)
    task_dir = os.path.join(tree, "codes", "config", case["task"])
    S = case["size"]
    rng = np.random.RandomState(0)
    for split, n in (("train", 4), ("val", 2)):
        for kind in ("GT", "LQ"):
            os.makedirs(os.path.join(tree, "data", split, kind))
        for i in range(n):   # smooth images, so that PSNR is not dominated by the sampler's noise floor
            gt = cv2.resize((rng.rand(S // 8, S // 8, 3) * 255).astype(np.uint8), (S, S), interpolation=cv2.INTER_CUBIC)
            lq = np.clip(gt.astype(np.int32) + rng.randint(-25, 25, gt.shape), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(tree, "data", split, "GT", "%d.png" % i), gt)
            cv2.imwrite(os.path.join(tree, "data", split, "LQ", "%d.png" % i), lq)
    opt = yaml.safe_load(open(os.path.join(task_dir, case["yml"])))
    opt["name"] = "train_ab"
    opt["use_tb_logger"] = True      # train.py:315 closes the tensorboard logger unconditionally
    opt["sde"]["T"] = 12
    for phase in ("train", "val"):
        d = opt["datasets"][phase]
        d["dataroot_GT"] = os.path.join(tree, "data", phase, "GT")
        if "dataroot_LQ" in d:
            d["dataroot_LQ"] = os.path.join(tree, "data", phase, "LQ")
    tr = opt["datasets"]["train"]
    # train.py leaves Python's `random` unseeded (train.py:75): only a crop as large as the image and no flips / rotations
    # make the dataset's draws (LQGT_dataset.py:137-152) return the same patches in both arms
    tr.update(n_workers=0, batch_size=2, GT_size=S, use_flip=False, use_rot=False, use_swap=False)
    if "LR_size" in tr:
        tr["LR_size"] = S
    opt["network_G"]["setting"] = dict(case["net"])
    opt["train"].update(niter=NITER, val_freq=VAL_FREQ)
    opt["logger"] = dict(print_freq=1, save_checkpoint_freq=1000)
    opt["path"]["pretrain_model_G"] = None
    yml = os.path.join(tree, "train_ab.yml")
    yaml.safe_dump(opt, open(yml, "w"), sort_keys=False)
    open(os.path.join(tree, "driver.py"), "w").write(DRIVER)
    return task_dir, yml, opt


def _run_arm(tree, task_dir, yml, launcher, env_extra, log):
    env = dict(os.environ)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    env["NVIDIA_TF32_OVERRIDE"] = "0"      # both arms train the same fp32 autograd network
    env.update(env_extra)
    out_json = os.path.join(tree, "driver.json")
    cmd = [sys.executable, os.path.join(tree, "driver.py"), ROOT, out_json] + launcher + \
        [os.path.join(task_dir, "train.py"), "-opt=" + yml]
    p = subprocess.run(cmd, cwd=task_dir, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    open(log, "w").write(p.stdout)
    assert p.returncode == 0, p.stdout[-4000:]
    psnrs = [float(line.rsplit("psnr:", 1)[1]) for line in p.stdout.splitlines() if line.startswith("<epoch:") and "psnr:" in line]
    return psnrs, json.load(open(out_json))


def _checkpoint(tree, task):
    import torch
    return torch.load(os.path.join(tree, "experiments", task, "train_ab", "models", "latest_G.pth"))


PSNR_BOUND_DB = 0.05


@pytest.mark.parametrize("case", sorted(CASES))
def test_reference_train_py_runs_unchanged(tmp_path, case):
    _need_gpu_and_ref()
    import torch
    c = CASES[case]
    arms = {}
    for arm, launcher, env in (("native", ["--seed", "7"], {"IRSDE_B200_PRECISION": "fp32"}),
                               ("reference", ["--seed", "7", "--reference"], {})):
        tree = str(tmp_path / arm)
        task_dir, yml, opt = _write_tree(tree, c)
        psnrs, info = _run_arm(tree, task_dir, yml, launcher, env, str(tmp_path / (arm + ".log")))
        arms[arm] = dict(tree=tree, psnrs=psnrs, info=info)
    nat, ref = arms["native"], arms["reference"]
    print("%s on %s" % (case, _card()))
    for arm, a in arms.items():
        print("  %-9s val PSNR %s; per validation pass: %s" % (arm, ["%.4f" % v for v in a["psnrs"]], [
            "%.1f ms, torch peak %.0f MiB, device used %.0f MiB" % (p["seconds"] * 1e3, p["torch_peak_bytes"] / 2 ** 20,
                                                                    p["device_used_bytes"] / 2 ** 20)
            for p in a["info"]["passes"]]))
    n_val = NITER // VAL_FREQ
    assert len(nat["psnrs"]) == len(ref["psnrs"]) == n_val and len(nat["info"]["passes"]) == n_val
    worst = max(abs(a - b) for a, b in zip(nat["psnrs"], ref["psnrs"]))
    print("  max |PSNR native - reference| = %.2e dB (bound %.2f dB)" % (worst, PSNR_BOUND_DB))
    assert worst <= PSNR_BOUND_DB
    # validation ran on the native kernels, with one weight upload per validation pass; the reference arm adopted nothing
    sh = [s for s in nat["info"]["shadows"] if s is not None]
    assert len(sh) == 1 and sh[0]["launches"] > 0 and sh[0]["uploads"] == n_val, nat["info"]["shadows"]
    assert sh[0]["cls"] == ("ConditionalUNet" if "ir-sde" in case else
                            "DenoisingNAFNet" if c["task"] == "denoising-sde" else "ConditionalNAFNet")
    assert sh[0]["latent"] == (c["task"] == "latent-dehazing")
    assert ref["info"]["shadows"] == []
    # training stayed on the reference's autograd path (the checkpoints agree up to cuDNN's non-deterministic backward,
    # which moves a parameter by at most ~lr per step for Lion's sign update and Adam's normalised one), and no shadow
    # leaked into the saved state dict
    a, b = _checkpoint(nat["tree"], c["task"]), _checkpoint(ref["tree"], c["task"])
    assert list(a) == list(b)
    lr = float(opt["train"]["lr_G"])
    diff = max((a[k].float() - b[k].float()).abs().max().item() for k in a)
    print("  final G checkpoints: max |native - reference| = %.2e (bound 2 * lr * niter = %.2e)" % (diff, 2 * lr * NITER))
    assert diff <= 2 * lr * NITER


def test_reference_train_py_bf16_validation(tmp_path):
    """The native arm in bf16 (the perf precision) on the deraining refusion case: the run completes with finite PSNR."""
    _need_gpu_and_ref()
    c = CASES["deraining-refusion"]
    tree = str(tmp_path / "native")
    task_dir, yml, _ = _write_tree(tree, c)
    psnrs, info = _run_arm(tree, task_dir, yml, ["--seed", "7"], {"IRSDE_B200_PRECISION": "bf16"}, str(tmp_path / "bf16.log"))
    print("bf16 native arm on %s: val PSNR %s, per pass %s" % (_card(), psnrs, ["%.1f ms" % (p["seconds"] * 1e3)
                                                                               for p in info["passes"]]))
    assert len(psnrs) == NITER // VAL_FREQ and all(math.isfinite(v) for v in psnrs)
    sh = [s for s in info["shadows"] if s is not None]
    assert len(sh) == 1 and sh[0]["launches"] > 0
