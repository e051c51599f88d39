"""The batched one-sided copy kernel (rmaCopyManyKernel, behind put_many /
get_many and MPI_Rput / MPI_Rget) is Hopper code that moves the aligned
middle of a copy in 128-bit global loads and stores and keeps everything in
registers (checked from the SASS, no GPU needed)."""

import re
import shutil
import subprocess

import pytest

from faabric_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
KERNEL = "_ZN2fb17rmaCopyManyKernelENS_11RmaCopyArgsE"

pytestmark = pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not installed")


def _run(*args):
    r = subprocess.run([CUOBJDUMP, *args, str(_lib.lib_path())], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    return r.stdout


def test_copy_kernel_is_sm_90a_with_128_bit_global_accesses(native_lib):
    sass = _run("-sass", "-fun", KERNEL)
    assert "arch = sm_90a" in sass, sass[:400]
    ops = set(re.findall(r"\b([A-Z][A-Z0-9_]*(?:\.[A-Z0-9_]+)*)\b", sass))
    assert "LDG.E.128" in ops and "STG.E.128" in ops, sorted(o for o in ops if o.startswith(("LDG", "STG")))
    # and the narrower widths of misaligned copies
    for w in ("LDG.E.64", "STG.E.64", "LDG.E", "STG.E", "LDG.E.U16", "STG.E.U16", "LDG.E.U8", "STG.E.U8"):
        assert w in ops, w
    assert not any(o.startswith(("LDL", "STL")) for o in ops), "local-memory traffic"


def test_copy_kernel_does_not_spill(native_lib):
    usage = _run("-res-usage")
    m = re.search(re.escape(KERNEL) + r":\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", usage)
    assert m, "rmaCopyManyKernel missing from the library"
    reg, stack, _, local = (int(x) for x in m.groups())
    # two 256-thread CTAs per SM (its launch bounds) need at most 128 registers
    assert reg <= 128 and stack == 0 and local == 0, m.group(0)
