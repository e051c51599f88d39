"""The grouped gather and scatter kernels (groupGatherKernel and
groupScatterKernel, behind gather_many / scatter_many and MPI_Igather /
MPI_Iscatter bursts) are Hopper code that keeps everything in registers
(checked from the SASS, no GPU needed)."""

import re
import shutil
import subprocess

import pytest

from faabric_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
KERNELS = ["_ZN2fb17groupGatherKernelILi", "_ZN2fb18groupScatterKernelILi"]
ARGS = "EEEvNS_9GroupArgsE"
NRS = [0, 1, 2, 4, 8]

pytestmark = pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not installed")


def _run(*args):
    r = subprocess.run([CUOBJDUMP, *args, str(_lib.lib_path())], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    return r.stdout


@pytest.mark.parametrize("nr", NRS)
@pytest.mark.parametrize("prefix", KERNELS, ids=["gather", "scatter"])
def test_kernel_is_sm90a_without_local_memory(native_lib, prefix, nr):
    sass = _run("-sass", "-fun", f"{prefix}{nr}{ARGS}")
    assert "arch = sm_90a" in sass, sass[:400]
    ops = set(re.findall(r"\b([A-Z][A-Z0-9_]*(?:\.[A-Z0-9_]+)*)\b", sass))
    # 128-bit loads and stores where the user side is 16-byte aligned
    assert any(o.startswith("LDG.E.128") for o in ops) and any(o.startswith("STG.E.128") for o in ops), sorted(
        o for o in ops if o.startswith(("LDG", "STG"))
    )
    assert not any(o.startswith(("LDL", "STL")) for o in ops), "local-memory traffic"


@pytest.mark.parametrize("prefix", KERNELS, ids=["gather", "scatter"])
def test_no_instantiation_spills(native_lib, prefix):
    usage = _run("-res-usage")
    found = re.findall(re.escape(prefix) + r"\w+:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", usage)
    assert len(found) == len(NRS), len(found)
    # at most 128 registers: 512 threads per CTA stay resident
    for reg, stack, _, local in found:
        assert int(reg) <= 128 and int(stack) == 0 and int(local) == 0, (reg, stack, local)
