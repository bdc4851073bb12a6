"""Compile-output guard for the register budget of the tensor-core DQN learner (no GPU needed).

k_dqn_tc runs one CTA per SM with 225 KB of shared memory, so the L1 left beside it cannot hold the kernel's spill
frame and spill reloads reach L2; one inside a wgmma chain holds up every product issued after it.  These
tests read what build() left, like tests/test_dqn_tc_sass.py: no spill reload (LDL) between the first and the last HGMMA
of a chain (the HGMMA of one product, the last of which carries gsb0), spill stores (STL) there only as counted below,
and the spill bytes ptxas reports within the figures below.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "pearl_b200", "build.log")
LIB = os.path.join(ROOT, "pearl_b200", "libpearlb200.so")
# (spill stores, spill loads) in bytes per dW1s share NW, as ptxas reports them for sm_90a
MAX_SPILL = {64: (376, 428), 32: (480, 536), 16: (112, 124), 8: (88, 104)}
# local-memory accesses allowed inside the chains of one instantiation: ptxas computes the descriptors of a whole group of
# products before its first wgmma, and in the NW = 32 kernel that pushes one register pair out at the start of the dW2 chain
MAX_IN_CHAINS = {64: 0, 32: 1, 16: 0, 8: 0}


def _log():
    if not os.path.exists(LOG) or not os.path.exists(LIB):
        pytest.skip("build() has not been run: no pearl_b200/build.log / libpearlb200.so")
    return open(LOG).read()


def _instantiations(log):
    syms = sorted(set(re.findall(r"Compiling entry function '(\S*k_dqn_tcILi(\d+)E\S*)'", log)))
    assert sorted(int(nw) for _, nw in syms) == [8, 16, 32, 64], f"expected the four k_dqn_tc instantiations, found {syms}"
    return syms


def _chains(sass):
    """Instruction lists from the first to the last HGMMA of each product (its last HGMMA carries gsb0)."""
    ins = [line for line in sass.splitlines() if re.search(r"/\*[0-9a-f]{4,}\*/\s+\S", line)]
    chains, start = [], None
    for k, line in enumerate(ins):
        if re.search(r"\bHGMMA\.", line):
            if start is None:
                start = k
            if "gsb0" in line:
                chains.append(ins[start:k + 1])
                start = None
    return chains


def test_k_dqn_tc_spill_bytes():
    log = _log()
    for sym, nw in _instantiations(log):
        m = re.search(re.escape(sym) + r"\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
        assert m, f"no ptxas function properties for {sym} in build.log"
        stores, loads = int(m.group(1)), int(m.group(2))
        max_st, max_ld = MAX_SPILL[int(nw)]
        assert stores <= max_st and loads <= max_ld, (
            f"k_dqn_tc<{nw}>: {stores} B spill stores / {loads} B spill loads, at most {max_st} / {max_ld} expected")


def test_k_dqn_tc_no_spill_inside_chains():
    log = _log()
    cuobjdump = shutil.which("cuobjdump") or ("/usr/local/cuda/bin/cuobjdump" if os.path.exists("/usr/local/cuda/bin/cuobjdump") else None)
    if cuobjdump is None:
        pytest.skip("cuobjdump is not on the path")
    for sym, nw in _instantiations(log):
        sass = subprocess.run([cuobjdump, "-sass", "-fun", sym, LIB], capture_output=True, text=True, check=True).stdout
        chains = _chains(sass)
        assert chains, f"k_dqn_tc<{nw}>: no HGMMA found"
        spills = [x.strip() for c in chains for x in c if re.search(r"\b(LDL|STL)\b", x)]
        assert not any(re.search(r"\bLDL\b", x) for x in spills), f"k_dqn_tc<{nw}>: spill reloads inside a chain:\n" + "\n".join(spills[:10])
        assert len(spills) <= MAX_IN_CHAINS[int(nw)], (f"k_dqn_tc<{nw}>: {len(spills)} spill stores inside the chains, at most "
                                                       f"{MAX_IN_CHAINS[int(nw)]} expected:\n" + "\n".join(spills[:10]))
