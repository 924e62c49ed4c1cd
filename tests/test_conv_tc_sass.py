"""CPU-only guard on the compiled tensor-core conv: every wgmma of conv_tc_persist_kernel must stay asynchronous.

ptxas serializes all wgmma instructions of a kernel whose wgmma window crosses a function call (warning C7510): each
HGMMA is then followed by `WARPGROUP.DEPBAR.LE gsb0, 0x0` and the K loop never keeps a group in flight.  A single printf
on the pipeline's wait path is enough to cause this, so the test compiles conv_tc.cu for sm_90a exactly as build.py
does and checks the ptxas log and the SASS of every instantiation.
"""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "image-restoration-sde_b200")


def _build_module():
    spec = importlib.util.spec_from_file_location("irsde_b200_build_sass", os.path.join(PKG, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _split_functions(sass):
    """{mangled name: [instruction text, ...]} for every function in a cuobjdump -sass listing."""
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if m and cur is not None:
            cur.append(m.group(1))
    return funcs


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    b = _build_module()
    nvcc = b.NVCC if os.path.isfile(b.NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.isfile(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = tmp_path_factory.mktemp("conv_tc_sass")
    obj = str(out / "conv_tc.o")
    r = subprocess.run([nvcc] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(b.CSRC, "conv_tc.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    s = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True)
    kernels = {k: v for k, v in _split_functions(s.stdout).items() if "conv_tc_persist_kernel" in k}
    assert kernels, "no conv_tc_persist_kernel instantiation in the object"
    return r.stdout + r.stderr, kernels


def _mode(name):
    m = re.search(r"conv_tc_persist_kernelILi(\d+)ELi(\d+)ELi(\d+)E", name)
    assert m, name
    return int(m.group(2))


def test_ptxas_does_not_serialize_wgmma(compiled):
    log, _ = compiled
    assert "C7510" not in log, "\n".join(l for l in log.splitlines() if "C7510" in l or "serialized" in l)


def test_no_external_call(compiled):
    _, kernels = compiled
    bad = {k: [i for i in ins if "CALL.ABS" in i] for k, ins in kernels.items()}
    assert not {k: v for k, v in bad.items() if v}


def test_k_loop_keeps_one_wgmma_group_in_flight(compiled):
    _, kernels = compiled
    assert {0, 2, 3} <= {_mode(k) for k in kernels}  # per-tap, ROWS and fp32x3 instantiations are all checked
    for name, ins in kernels.items():
        assert any(re.match(r"HGMMA\.", i) for i in ins), name
        # the K loop retires all but the newest group: wgmma.wait_group 1
        assert any("WARPGROUP.DEPBAR.LE gsb0, 0x1" in i for i in ins), name
        # a wait for zero groups directly behind an MMA is the serialized form; the only full wait is the drain before the
        # epilogue, which follows the loop's branch rather than an HGMMA
        for a, b in zip(ins, ins[1:]):
            assert not (a.startswith("HGMMA.") and "WARPGROUP.DEPBAR.LE gsb0, 0x0" in b), (name, a, b)
