"""Stage the UNMODIFIED reference (Algolzw/image-restoration-sde) under oracle/_ref/.

The reference is plain Python with no package metadata, so the files its sampling path needs are copied verbatim:
Python sources and YAMLs of `codes/utils`, `codes/data` and three task directories, plus the one trained checkpoint and
the one sample image that tests/test_oracle_golden.py::test_latent_unet_oracle_real_checkpoint reads.  oracle/_ref/ is
git-ignored (never part of this repository's history).  Called by __graft_entry__.build(); a no-op where the reference
checkout (SRC) does not exist, so a tree built next to the reference carries it along.

Used only by: `bench.py --impl reference` (the reference's own IRSDE + ConditionalUNet, CPU or CUDA eager),
tests/test_gpu_dropin.py (the reference's test.py run unchanged through `python -m irsde_b200.run`),
tests/test_host.py::test_launcher_patches_reference_tree and the real-checkpoint oracle test.
"""
import os
import shutil

SRC = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, "_ref")
TREES = ["codes/utils", "codes/data", "codes/config/deraining", "codes/config/denoising-sde", "codes/config/latent-dehazing"]
KEEP_EXT = (".py", ".yml", ".yaml", ".sh", ".txt")
FILES = ["codes/config/latent-dehazing/pretrained_models/latent-dehazing.pth", "images/1.png", "LICENSE", "requirements.txt"]


def stage(force=False):
    if not os.path.isdir(SRC):
        return os.path.isdir(DST)
    stamp = os.path.join(DST, ".staged")
    if os.path.exists(stamp) and not force:
        return True
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    n = 0
    for tree in TREES:
        for root, dirs, files in os.walk(os.path.join(SRC, tree)):
            dirs[:] = [d for d in dirs if d != "__pycache__"]
            for f in files:
                if not f.endswith(KEEP_EXT):
                    continue
                src = os.path.join(root, f)
                if os.path.getsize(src) > (1 << 20):
                    continue
                dst = os.path.join(DST, os.path.relpath(src, SRC))
                os.makedirs(os.path.dirname(dst), exist_ok=True)
                shutil.copyfile(src, dst)
                n += 1
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
        f.write("files=%d\ncommit=%s\n" % (n, commit))
    return True


if __name__ == "__main__":
    print(stage(force=True), open(os.path.join(DST, ".staged")).read())
