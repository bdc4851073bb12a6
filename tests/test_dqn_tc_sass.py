"""Compile-output guard for the tensor-core DQN learner (no GPU needed).

ptxas decides per kernel whether its wgmma instructions may pipeline.  One obstacle anywhere in k_dqn_tc (a function
call, a wgmma under a branch, a chain that does not fit in the registers) makes it wait after EVERY wgmma of the
kernel, which puts each 24-instruction 3xTF32 product at instruction latency.  These tests read what build() left:
the -Xptxas -v log and the SASS of every k_dqn_tc instantiation.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "pearl_b200", "build.log")
LIB = os.path.join(ROOT, "pearl_b200", "libpearlb200.so")
# wgmma.wait_group sites executed by k_dqn_tc: layer 1 (inlined twice: phase T and phase O), the phase-T action loop,
# online layer 2, dH1, and the two weight-gradient passes
WAIT_SITES = 7


def _log():
    if not os.path.exists(LOG) or not os.path.exists(LIB):
        pytest.skip("build() has not been run: no pearl_b200/build.log / libpearlb200.so")
    return open(LOG).read()


def _symbols(log):
    syms = sorted(set(re.findall(r"Compiling entry function '(\S*k_dqn_tc\S*)'", log)))
    assert len(syms) == 4, f"expected the four k_dqn_tc instantiations (dW1s shares 8/16/32/64), found {syms}"
    return syms


def test_k_dqn_tc_wgmma_not_serialised():
    log = _log()
    for sym in _symbols(log):
        warnings = [line for line in log.splitlines() if re.search(r"\(C75\d\d\)", line) and sym in line]
        assert not warnings, "ptxas serialises the wgmma of " + sym + ":\n" + "\n".join(warnings)


def test_k_dqn_tc_sass_chains_unbroken():
    log = _log()
    cuobjdump = shutil.which("cuobjdump") or ("/usr/local/cuda/bin/cuobjdump" if os.path.exists("/usr/local/cuda/bin/cuobjdump") else None)
    if cuobjdump is None:
        pytest.skip("cuobjdump is not on the path")
    for sym in _symbols(log):
        sass = subprocess.run([cuobjdump, "-sass", "-fun", sym, LIB], capture_output=True, text=True, check=True).stdout
        hgmma = len(re.findall(r"\bHGMMA\.", sass))
        depbar = len(re.findall(r"WARPGROUP\.DEPBAR", sass))
        assert hgmma >= 24 * WAIT_SITES, f"{sym}: only {hgmma} HGMMA"
        assert depbar <= WAIT_SITES, f"{sym}: {depbar} WARPGROUP.DEPBAR for {hgmma} HGMMA (at most {WAIT_SITES} expected)"
