"""Register and spill guard for the banded engine (csrc/engine.cuh).

Every engine_kernel instance is compiled under __launch_bounds__(256, 6), which leaves 40 registers per thread; a
change to the slot loops that needs more makes ptxas spill instead of failing.  This test compiles the translation
units that instantiate the engine for sm_90a with `-Xptxas -v` and checks each instance's registers and spill stores
against the figures recorded in DESIGN.md section 4.  No GPU is needed; it is skipped where nvcc is absent."""
import os
import re
import shutil
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rapidcfd-dev_b200", "csrc")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ENGINE_UNITS = ["ldu.cu", "solvers.cu", "comm.cu", "layout.cu"]

MAX_REGISTERS = 40
# spill stores (bytes) allowed per (operator, face stream): the face-stream owner pass keeps a group of three
# coefficient and template-word loads in flight, which costs a few bytes of spill in the operators with the most state;
# every instance not listed must not spill at all
SPILL_STORE_CEILING = {
    ("PcgAmulOp", False): 52,
    ("PcgAmulOp", True): 60,
    ("AmulOp", True): 12,
    ("JacobiOp", True): 12,
    ("ResidualOp", True): 12,
    ("OffDiagOp", True): 12,
}


def _compile(unit, out_dir):
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--extended-lambda",
           "-Xcompiler", "-fPIC,-fopenmp", "-Xptxas", "-v", "-c", "-o", os.path.join(out_dir, unit + ".o"), unit]
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    r = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def _engine_instances(log):
    """{mangled name: (registers, spill store bytes)} of the engine_kernel instances in one ptxas -v log"""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m and cur:
            out.setdefault(cur, [0, 0])[1] = int(m.group(1))
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            out.setdefault(cur, [0, 0])[0] = int(m.group(1))
            cur = None
    return {k: tuple(v) for k, v in out.items() if "13engine_kernel" in k}


def _op_and_stream(mangled):
    """operator name and face-stream flag of _Z13engine_kernelI<len><Op>...ELb<FS>EEv9LayoutDev..."""
    m = re.match(r"_Z13engine_kernelI(\d+)", mangled)
    n = int(m.group(1))
    op = mangled[m.end():m.end() + n]
    fs = re.search(r"Lb([01])EEv9LayoutDev", mangled)
    return op, fs.group(1) == "1"


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_engine_kernels_fit_40_registers_without_new_spills():
    with tempfile.TemporaryDirectory() as tmp, ThreadPoolExecutor(len(ENGINE_UNITS)) as ex:
        logs = list(ex.map(lambda u: _compile(u, tmp), ENGINE_UNITS))
    inst = {}
    for log in logs:
        inst.update(_engine_instances(log))
    assert len(inst) >= 30, f"expected every engine_kernel instance, found {len(inst)}"
    seen_fs = set()
    bad = []
    for name, (regs, spill) in sorted(inst.items()):
        op, fs = _op_and_stream(name)
        seen_fs.add(fs)
        ceiling = SPILL_STORE_CEILING.get((op, fs), 0)
        if regs > MAX_REGISTERS or spill > ceiling:
            bad.append(f"{op} face_stream={fs}: {regs} registers, {spill} B spill stores (ceiling {ceiling} B)")
    assert seen_fs == {False, True}
    assert not bad, "\n".join(bad)
