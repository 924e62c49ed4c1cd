"""Stage the UNMODIFIED reference (Algolzw/image-restoration-sde) under oracle/_ref/.

The reference is plain Python with no package metadata, so the files its sampling path needs are copied verbatim:
Python sources and YAMLs of `codes/utils`, `codes/data` and three task directories, the `options/` YAMLs of every task
directory, plus the one trained checkpoint and the one sample image that
tests/test_oracle_golden.py::test_latent_unet_oracle_real_checkpoint reads.  The `.staged` stamp records TREES: a
staging made from another list is redone.  oracle/_ref/ is
git-ignored (never part of this repository's history).  Called by __graft_entry__.build(); a no-op where the reference
checkout (SRC) does not exist, so a tree built next to the reference carries it along.

Used only by: `bench.py --impl reference` (the reference's own IRSDE + ConditionalUNet, CPU or CUDA eager),
tests/test_gpu_dropin.py (the reference's test.py run unchanged through `python -m irsde_b200.run`),
tests/test_host.py::test_launcher_patches_reference_tree, the real-checkpoint oracle test and the coverage guard of
tests/test_gpu_task_networks.py (every network a task's test options build).
"""
import glob
import os
import shutil

SRC = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, "_ref")
TREES = ["codes/utils", "codes/data", "codes/config/deraining", "codes/config/denoising-sde", "codes/config/latent-dehazing",
         "codes/config/*/options"]
KEEP_EXT = (".py", ".yml", ".yaml", ".sh", ".txt")
FILES = ["codes/config/latent-dehazing/pretrained_models/latent-dehazing.pth", "images/1.png", "LICENSE", "requirements.txt"]


def stage(force=False):
    if not os.path.isdir(SRC):
        return os.path.isdir(DST)
    stamp = os.path.join(DST, ".staged")
    trees = "trees=%s\n" % ",".join(TREES)
    if os.path.exists(stamp) and not force:
        with open(stamp) as f:
            if trees in f.read().splitlines(keepends=True):
                return True
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    copied = set()   # a task's options/ also lies inside the task trees staged whole
    for tree in sorted({d for pattern in TREES for d in glob.glob(os.path.join(SRC, pattern))}):
        for root, dirs, files in os.walk(tree):
            dirs[:] = [d for d in dirs if d != "__pycache__"]
            for f in files:
                src = os.path.join(root, f)
                if not f.endswith(KEEP_EXT) or src in copied or os.path.getsize(src) > (1 << 20):
                    continue
                dst = os.path.join(DST, os.path.relpath(src, SRC))
                os.makedirs(os.path.dirname(dst), exist_ok=True)
                shutil.copyfile(src, dst)
                copied.add(src)
    for extra in FILES:
        if os.path.exists(os.path.join(SRC, extra)):
            dst = os.path.join(DST, extra)
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            shutil.copyfile(os.path.join(SRC, extra), dst)
    commit = ""
    try:
        import json
        commit = json.load(open(os.path.join(SRC, ".SUBMODULES.json"))).get("commit", "")
    except Exception:
        pass
    with open(stamp, "w") as f:
        f.write("files=%d\ncommit=%s\n%s" % (len(copied), commit, trees))
    return True


if __name__ == "__main__":
    print(stage(force=True), open(os.path.join(DST, ".staged")).read())
