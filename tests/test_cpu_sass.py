"""The built library is Hopper code: sm_90a cubins only, and the kernels
contain the instructions the design depends on (checked from the SASS, no GPU
needed).  Mnemonics: profiles/sass/MNEMONICS.md."""

import re
import shutil
import subprocess

import pytest

from faabric_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

pytestmark = pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not installed")


def _sass(function: str) -> str:
    r = subprocess.run([CUOBJDUMP, "-sass", "-fun", function, str(_lib.lib_path())], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    return r.stdout


def _mnemonics(sass: str) -> set:
    return set(re.findall(r"\b([A-Z][A-Z0-9_]*(?:\.[A-Z0-9_]+)*)\b", sass))


def test_only_sm_90a_cubins_are_embedded(native_lib):
    r = subprocess.run([CUOBJDUMP, "-lelf", str(_lib.lib_path())], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    elfs = re.findall(r"ELF file\s+\d+:\s+(\S+)", r.stdout)
    assert len(elfs) >= 6, r.stdout
    assert all(e.endswith(".sm_90a.cubin") for e in elfs), elfs
    # no PTX for a JIT fallback on another architecture either
    r = subprocess.run([CUOBJDUMP, "-lptx", str(_lib.lib_path())], capture_output=True, text=True, timeout=120)
    assert "PTX file" not in r.stdout, r.stdout


def test_bulk_copy_kernel_uses_tma_and_mbarriers(native_lib):
    ops = _mnemonics(_sass("_ZN2fb14moveBulkKernelENS_8MoveArgsE"))
    # cp.async.bulk global->shared and shared->global, mbarrier arrive/try_wait
    assert "UBLKCP.S.G" in ops and "UBLKCP.G.S" in ops, sorted(o for o in ops if o.startswith("UBLKCP"))
    assert any(o.startswith("SYNCS.ARRIVE") for o in ops)
    assert any(o.startswith("SYNCS.PHASECHK") for o in ops)


def test_nvls_kernel_reduces_in_the_switch(native_lib):
    ops = _mnemonics(_sass("_ZN2fb10nvlsKernelILi0EEEvNS_8NvlsArgsE"))
    # multimem.ld_reduce / multimem.st
    assert any(o.startswith("LDGMC") for o in ops), sorted(ops)[:40]
    assert any(o.startswith("STG") or o.startswith("STGMC") for o in ops)


def test_peer_loads_are_system_scope_and_vectorised(native_lib):
    r = subprocess.run([CUOBJDUMP, "-sass", str(_lib.lib_path())], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0
    # flag polling at .sys scope and 128-bit data movement over NVLink
    assert r.stdout.count("LDG.E.STRONG.SYS") > 100
    assert r.stdout.count("LDG.E.128") > 100
    assert "STG.E.128" in r.stdout


def test_kernels_fit_their_launch_bounds_without_spilling(native_lib):
    """Resource usage straight from the cubins: every kernel stays within 128
    registers (two 512-thread CTAs of the collectives per SM) and keeps at
    most a few words on the stack."""
    r = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.lib_path())], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    usage = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", r.stdout)
    assert len(usage) > 500, len(usage)
    assert max(int(u[1]) for u in usage) <= 128
    assert max(int(u[2]) for u in usage) <= 64
    assert all(int(u[4]) == 0 for u in usage)
    # the hot int32 SUM all-reduce (headline dtype) needs few registers
    hot = [u for u in usage if "llAllReduceKernel" in u[0]]
    assert hot and max(int(u[1]) for u in hot) <= 64
