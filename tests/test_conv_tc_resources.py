"""CPU-only guard on the registers of the compiled tensor-core conv: no conv_tc_persist_kernel instantiation spills.

The bf16 epilogue works on the wgmma accumulator registers (up to 2 x 64 per thread in the ping-pong tiles, 128 at
BN = 256), so a change that makes ptxas spill shows up as local-memory traffic in every tile.  The test compiles conv_tc.cu
for sm_90a as build.py does, with -Xptxas -v, and checks every instantiation's spill counts; it also checks that no bf16
instantiation calls a subroutine (the fp32x3 ones keep the IEEE-division slow path, a call after the K loop).
"""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "image-restoration-sde_b200")
KERNEL = re.compile(r"conv_tc_persist_kernelILi(\d+)ELi(\d+)ELi(\d+)E")


def _build_module():
    spec = importlib.util.spec_from_file_location("irsde_b200_build_res", os.path.join(PKG, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    b = _build_module()
    nvcc = b.NVCC if os.path.isfile(b.NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.isfile(cuobjdump):
        pytest.skip("cuobjdump not available")
    obj = str(tmp_path_factory.mktemp("conv_tc_res") / "conv_tc.o")
    r = subprocess.run([nvcc] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(b.CSRC, "conv_tc.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    s = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True)
    return r.stdout + r.stderr, s.stdout


def _spills(log):
    """{(BN, MODE, EKT): (spill store bytes, spill load bytes)} of every conv_tc_persist_kernel entry in a ptxas -v log."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            k = KERNEL.search(m.group(1))
            cur = tuple(int(x) for x in k.groups()) if k else None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            out[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return out


def test_no_instantiation_spills(compiled):
    spills = _spills(compiled[0])
    assert len(spills) == 21, sorted(spills)
    bad = {k: v for k, v in spills.items() if v != (0, 0)}
    assert not bad, "conv_tc_persist_kernel<BN, MODE, EKT> instantiations that spill (store, load bytes): %s" % bad


def test_bf16_instantiations_make_no_call(compiled):
    calls, cur = {}, None
    for line in compiled[1].splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            k = KERNEL.search(m.group(1))
            cur = tuple(int(x) for x in k.groups()) if k else None
            if cur:
                calls.setdefault(cur, 0)
            continue
        if cur is not None and re.search(r"\bCALL\.", line):
            calls[cur] += 1
    assert len(calls) == 21, sorted(calls)
    bad = {k: n for k, n in calls.items() if k[1] != 3 and n}
    assert not bad, "bf16 instantiations with CALL instructions: %s" % bad
