"""The grouped neighbour v kernel (groupNeighborVKernel<A2A>, behind
neighbor_all_gather_v_many / neighbor_all_to_all_v_many and their plans) is
Hopper code that keeps everything in registers (checked from the SASS, no GPU
needed): both instantiations, and their resource usage."""

import re
import shutil
import subprocess

import pytest

from faabric_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
PREFIX = "_ZN2fb20groupNeighborVKernelILb"
KERNELS = {"all_gather_v": PREFIX + "0EEEvNS_9GroupArgsE", "all_to_all_v": PREFIX + "1EEEvNS_9GroupArgsE"}

pytestmark = pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not installed")


def _run(*args):
    r = subprocess.run([CUOBJDUMP, *args, str(_lib.lib_path())], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    return r.stdout


@pytest.mark.parametrize("kind", list(KERNELS))
def test_kernel_is_sm90a_without_local_memory(native_lib, kind):
    sass = _run("-sass", "-fun", KERNELS[kind])
    assert "arch = sm_90a" in sass, sass[:400]
    ops = set(re.findall(r"\b([A-Z][A-Z0-9_]*(?:\.[A-Z0-9_]+)*)\b", sass))
    # 128-bit loads and stores where both ends of a piece are 16-byte aligned
    assert any(o.startswith("LDG.E.128") for o in ops) and any(o.startswith("STG.E.128") for o in ops), sorted(
        o for o in ops if o.startswith(("LDG", "STG"))
    )
    assert not any(o.startswith(("LDL", "STL")) for o in ops), "local-memory traffic"


def test_every_instantiation_fits(native_lib):
    usage = _run("-res-usage")
    found = re.findall(re.escape(PREFIX) + r"(\d)\w+:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", usage)
    assert sorted(f[0] for f in found) == ["0", "1"], found
    # at most 128 registers: 512 threads per CTA stay resident
    for _, reg, stack, _, local in found:
        assert int(reg) <= 128 and int(stack) == 0 and int(local) == 0, (reg, stack, local)
