"""CPU-only guards on the compiled tensor-core conv.  The module compiles conv_tc.cu once for sm_90a, exactly as build.py
does plus -Xptxas -v, and every check reads that one object's ptxas log or its cuobjdump -sass listing:

* Every wgmma of conv_tc_persist_kernel stays asynchronous.  ptxas serializes all wgmma instructions of a kernel whose
  wgmma window crosses a function call (warning C7510): each HGMMA is then followed by `WARPGROUP.DEPBAR.LE gsb0, 0x0`
  and the K loop never keeps a group in flight.  A single printf on the pipeline's wait path is enough to cause this.
* No instantiation spills.  The bf16 epilogue works on the wgmma accumulator registers (up to 2 x 64 per thread in the
  ping-pong tiles, 128 at BN = 256), so a change that makes ptxas spill shows up as local-memory traffic in every tile.
* No bf16 instantiation calls a subroutine (the fp32x3 ones keep the IEEE-division slow path, a call after the K loop).
* The object holds exactly the instantiations that test_gpu_conv_epilogues.CASES name, one case at least for each.
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
    """(ptxas log, {(BN, MODE, EKT): [instruction text, ...]} of every conv_tc_persist_kernel instantiation)."""
    b = _build_module()
    nvcc = b.NVCC if os.path.isfile(b.NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.isfile(cuobjdump):
        pytest.skip("cuobjdump not available")
    obj = str(tmp_path_factory.mktemp("conv_tc_sass") / "conv_tc.o")
    r = subprocess.run([nvcc] + b.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(b.CSRC, "conv_tc.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    s = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True)
    kernels = {}
    for name, ins in _split_functions(s.stdout).items():
        k = KERNEL.search(name)
        if k:
            kernels[tuple(int(x) for x in k.groups())] = ins
    assert kernels, "no conv_tc_persist_kernel instantiation in the object"
    return r.stdout + r.stderr, kernels


def test_ptxas_does_not_serialize_wgmma(compiled):
    log, _ = compiled
    assert "C7510" not in log, "\n".join(l for l in log.splitlines() if "C7510" in l or "serialized" in l)


def test_no_external_call(compiled):
    _, kernels = compiled
    bad = {k: [i for i in ins if "CALL.ABS" in i] for k, ins in kernels.items()}
    assert not {k: v for k, v in bad.items() if v}


def test_k_loop_keeps_one_wgmma_group_in_flight(compiled):
    _, kernels = compiled
    assert {0, 2, 3} <= {k[1] for k in kernels}  # per-tap, ROWS and fp32x3 instantiations are all checked
    for name, ins in kernels.items():
        assert any(re.match(r"HGMMA\.", i) for i in ins), name
        # the K loop retires all but the newest group: wgmma.wait_group 1
        assert any("WARPGROUP.DEPBAR.LE gsb0, 0x1" in i for i in ins), name
        # a wait for zero groups directly behind an MMA is the serialized form; the only full wait is the drain before the
        # epilogue, which follows the loop's branch rather than an HGMMA
        for a, b in zip(ins, ins[1:]):
            assert not (a.startswith("HGMMA.") and "WARPGROUP.DEPBAR.LE gsb0, 0x0" in b), (name, a, b)


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
    calls = {k: sum(1 for i in ins if re.search(r"\bCALL\.", i)) for k, ins in compiled[1].items()}
    assert len(calls) == 21, sorted(calls)
    bad = {k: n for k, n in calls.items() if k[1] != 3 and n}
    assert not bad, "bf16 instantiations with CALL instructions: %s" % bad


def test_every_compiled_instantiation_has_a_case(compiled):
    from test_gpu_conv_epilogues import CASES
    instantiated = set(compiled[1])
    named = {c["expect"] for c in CASES if c["expect"] is not None}
    assert len(instantiated) == 21, sorted(instantiated)
    assert instantiated == named, ("without a case", sorted(instantiated - named), "not compiled", sorted(named - instantiated))
