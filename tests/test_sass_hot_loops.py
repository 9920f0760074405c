"""The window loops of the key-table and small-table kernels, read from the SASS of the built library (no GPU needed).

Each pass of those loops gathers one random 64-byte table point per lane and adds it to a Jacobian accumulator.  The point must
arrive as four 128-bit loads, not sixteen 32-bit ones: every lane of a warp reads a different point, so each load is a divergent
request.  And the accumulator must stay in registers: the exceptional case of the addition (H = 0) is an out-of-line call, and
nothing may go to local memory on the common path because of it."""
import os
import re
import shutil

import pytest

from util import pkg
from tools import sass_stalls

KERNELS = ["ecdsa_verify_cached_kernel", "ecdsa_verify_small_kernel"]


def _cuobjdump():
    for d in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "bin", "cuobjdump")):
            return os.path.join(d, "bin", "cuobjdump")
    return shutil.which("cuobjdump")


@pytest.fixture(scope="module")
def sass():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump is not installed")
    b = pkg().binding
    if not os.path.exists(b.LIB_PATH):
        if shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"):
            pytest.skip("nvcc is not installed")
        b.build()
    return sass_stalls.dump(b.LIB_PATH, tool)


def window_loop(ins):
    """The instructions of the largest innermost loop: [target, back-branch] of a backward BRA that holds no other backward BRA."""
    loops = []
    for addr, text, _ in ins:
        if sass_stalls.opcode(text) == "BRA":
            target = int(re.search(r"(0x[0-9a-f]+)\s*$", text).group(1), 16)
            if target <= addr:
                loops.append((target, addr))
    inner = [l for l in loops if not any(o != l and l[0] <= o[0] and o[1] <= l[1] for o in loops)]
    assert inner, "no loop found"
    lo, hi = max(inner, key=lambda l: l[1] - l[0])
    return [(addr, text) for addr, text, _ in ins if lo <= addr <= hi]


@pytest.mark.parametrize("kernel", KERNELS)
def test_window_loop_memory_path(sass, kernel):
    ins = sass_stalls.parse(sass, kernel)
    assert ins, "%s is not in the library" % kernel
    body = window_loop(ins)
    # the body is the whole expanded addition: a loop of a few dozen instructions would be some other loop
    assert len(body) > 1000, (kernel, len(body))
    ops = [(hex(a), sass_stalls.opcode(t)) for a, t in body]
    gathers = [(a, op) for a, op in ops if op.startswith("LDG")]
    assert [op.split(".")[:3] for _, op in gathers] == [["LDG", "E", "128"]] * 4, (kernel, gathers)
    local = [(a, op) for a, op in ops if op.startswith(("STL", "LDL"))]
    assert not local, (kernel, local)
