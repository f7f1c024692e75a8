"""CPU: the compiled order of the wgmma attention kernel (cuobjdump -sass of the built library, no GPU needed).

A consumer warpgroup issues S_j = Q K_j^T together with P_{j-1} V_{j-1}, waits for S_j only (WARPGROUP.DEPBAR.LE gsb0,
0x1), runs the softmax of tile j, and only then waits for P_{j-1} V_{j-1} (WARPGROUP.DEPBAR.LE gsb0, 0x0).  ptxas is
free to schedule that second wait above the softmax, which would leave nothing overlapping the MMAs; every instantiation
of the kernel must keep exponentials (MUFU.EX2) between the two waits."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "vista_slam_b200", "csrc", "libsta_b200.so")


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None and os.path.exists("/usr/local/cuda/bin/cuobjdump"):
        exe = "/usr/local/cuda/bin/cuobjdump"
    return exe


def _attention_kernels():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump (CUDA toolkit) not found")
    assert os.path.exists(LIB), "libsta_b200.so is not built (python -m vista_slam_b200.build)"
    sass = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    kernels = {}
    name = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "attention_fwd_kernel" in m.group(1) else None
            if name:
                kernels[name] = []
            continue
        if name is None:
            continue
        if "MUFU.EX2" in line:
            kernels[name].append("ex2")
        elif re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", line):
            kernels[name].append("wait1")
        elif re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", line):
            kernels[name].append("wait0")
    return kernels


def test_softmax_runs_between_the_two_waits_in_every_instantiation():
    kernels = _attention_kernels()
    assert len(kernels) == 4, sorted(kernels)  # (1 or 2 consumer warpgroups) x (<= 16-key tail or not)
    for name, seq in kernels.items():
        waits = [i for i, tok in enumerate(seq) if tok == "wait1"]
        assert waits, "%s: no wait for S alone (wgmma_wait<1>)" % name
        for i in waits:
            nxt = seq.index("wait0", i)
            n_ex2 = seq[i:nxt].count("ex2")
            assert n_ex2 >= 10, "%s: %d MUFU.EX2 between the wait for S and the wait for P V" % (name, n_ex2)
