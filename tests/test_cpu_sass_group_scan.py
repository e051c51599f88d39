"""The grouped scan kernels (groupScanKernel<VR, NR>, behind scan_many /
scan_group and MPI_Iscan / MPI_Iexscan bursts; one template serves the scan
and the exscan) are Hopper code that keeps everything in registers (checked
from the SASS, no GPU needed): a representative reduction of each family at
every NR, and the resource usage of every instantiation."""

import re
import shutil
import subprocess

import pytest

from faabric_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
PREFIX = "_ZN2fb15groupScanKernelINS_9VecReduceI"
NRS = [0, 1, 2, 4, 8]
# VecReduce<T, OP, PAIR> of f32 sum, bf16 sum, i64 max, u8 bxor and f64_i32
# maxloc (as the kernels number the ops: max 0, sum 2, maxloc 8, bxor 11)
VRS = {
    "f32_sum": "fLi2ELb0EEELi{nr}EEEvNS_9GroupArgsE",
    "bf16_sum": "13__nv_bfloat16Li2ELb0EEELi{nr}EEEvNS_9GroupArgsE",
    "i64_max": "lLi0ELb0EEELi{nr}EEEvNS_9GroupArgsE",
    "u8_bxor": "hLi11ELb0EEELi{nr}EEEvNS_9GroupArgsE",
    "f64_i32_maxloc": "dLi8ELb1EEELi{nr}EEEvNS_9GroupArgsE",
}
# the grouped reduce-scatter kernel exists for every reduction the device has
RS_PREFIX = "_ZN2fb24groupReduceScatterKernelINS_9VecReduceI"

pytestmark = pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not installed")


def _run(*args):
    r = subprocess.run([CUOBJDUMP, *args, str(_lib.lib_path())], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    return r.stdout


@pytest.mark.parametrize("nr", NRS)
@pytest.mark.parametrize("vr", list(VRS))
def test_kernel_is_sm90a_without_local_memory(native_lib, vr, nr):
    sass = _run("-sass", "-fun", PREFIX + VRS[vr].format(nr=nr))
    assert "arch = sm_90a" in sass, sass[:400]
    ops = set(re.findall(r"\b([A-Z][A-Z0-9_]*(?:\.[A-Z0-9_]+)*)\b", sass))
    # 128-bit loads and stores: the staged slices are 16-byte aligned
    assert any(o.startswith("LDG.E.128") for o in ops) and any(o.startswith("STG.E.128") for o in ops), sorted(
        o for o in ops if o.startswith(("LDG", "STG"))
    )
    assert not any(o.startswith(("LDL", "STL")) for o in ops), "local-memory traffic"


def test_every_instantiation_fits(native_lib):
    usage = _run("-res-usage")
    found = re.findall(re.escape(PREFIX) + r"\w+:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", usage)
    # every reduction the device has (one VecReduce per distinct (type, op)
    # kernel: signed and unsigned sums share one), at every NR, once: the
    # exclusive scan is a launch argument, not an instantiation
    vrs = set(re.findall(re.escape(RS_PREFIX) + r"(\w+?)Li\d+EEEvNS_9GroupArgsE", usage))
    ours = set(re.findall(re.escape(PREFIX) + r"(\w+?)Li\d+EEEvNS_9GroupArgsE", usage))
    assert ours == vrs and len(vrs) > 50, (len(ours), len(vrs))
    assert len(found) == len(vrs) * len(NRS), len(found)
    # at most 128 registers: 512 threads per CTA stay resident
    for reg, stack, _, local in found:
        assert int(reg) <= 128 and int(stack) == 0 and int(local) == 0, (reg, stack, local)
