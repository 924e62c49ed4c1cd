"""Build libirsde_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libirsde_b200.so")
SOURCES = ["engine.cu", "conv_simt.cu", "conv_tc.cu", "elementwise.cu", "attention.cu", "nafnet.cu", "imaging.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "-cudart", "static"]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "irsde_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def csrc_sha256():
    """Hash of the CUDA sources + the C header: names the build a bench line was measured on (BUILD_INFO)."""
    import hashlib
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh")):
            h.update(f.encode())
            h.update(open(os.path.join(CSRC, f), "rb").read())
    h.update(open(os.path.join(HERE, "..", "include", "irsde_b200.h"), "rb").read())
    return h.hexdigest()[:16]


def conv_tc_sha256(read=None):
    """Hash of the sources the tensor-core conv kernel compiles from (conv_tc.cu + common.cuh): tells whether two builds run
    the same conv kernel when only the other kernels changed."""
    import hashlib
    read = read or (lambda f: open(os.path.join(CSRC, f), "rb").read())
    h = hashlib.sha256()
    for f in ("common.cuh", "conv_tc.cu"):
        h.update(f.encode())
        h.update(read(f))
    return h.hexdigest()[:16]


def _write_build_info():
    try:
        commit = subprocess.run(["git", "-C", HERE, "rev-parse", "--short", "HEAD"], capture_output=True, text=True).stdout.strip()
        dirty = bool(subprocess.run(["git", "-C", HERE, "status", "--porcelain", "--", "csrc", "../include"], capture_output=True,
                                    text=True).stdout.strip())
    except Exception:
        commit, dirty = "", False
    if not commit:  # no git here (the GPU box ships without .git): keep the commit recorded when the library was built
        try:
            for line in open(os.path.join(HERE, "BUILD_INFO")):
                if line.startswith("commit="):
                    commit, dirty = line.strip()[7:].replace("+dirty", ""), "+dirty" in line
        except Exception:
            pass
    with open(os.path.join(HERE, "BUILD_INFO"), "w") as f:
        f.write("commit=%s%s\ncsrc_sha256=%s\nconv_tc_sha256=%s\n" % (commit or "unknown", "+dirty" if dirty else "", csrc_sha256(),
                                                                       conv_tc_sha256()))


def build(force=False, verbose=False):
    if not force and not _stale():
        _write_build_info()
        return LIB
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write("== %s ==\n%s\n" % (src, out))
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed building libirsde_b200.so")
    cmd = [NVCC, "-shared"] + FLAGS[:2] + ["-cudart", "static", "-o", LIB] + objs + ["-ldl", "-lpthread", "-lrt"]
    subprocess.check_call(cmd)
    _write_build_info()
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
