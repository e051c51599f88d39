"""The batched accumulate kernel (rmaAccumulateManyKernel, behind
accumulate_many and MPI_Raccumulate / MPI_Rget_accumulate bursts) is Hopper
code that keeps everything in registers, and applies integer and f64 sums
with native system-scope RED / ATOM instructions rather than CAS loops
(checked from the SASS, no GPU needed)."""

import re
import shutil
import subprocess

import pytest

from faabric_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
PREFIX = "_ZN2fb23rmaAccumulateManyKernelI"
ARGS = "EEEvNS_14RmaAccManyArgsE"
# (FbDtype code, FbOp code) -> the native add it must use
NATIVE_SUMS = {
    "i32": ((4, 2), "ADD.STRONG.SYS"),
    "i64": ((6, 2), "ADD.64.STRONG.SYS"),
    "f64": ((9, 2), "ADD.F64.RN.STRONG.SYS"),
}

pytestmark = pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not installed")


def _run(*args):
    r = subprocess.run([CUOBJDUMP, *args, str(_lib.lib_path())], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    return r.stdout


def _name(dt, op):
    return f"{PREFIX}Li{dt}ELi{op}{ARGS}"


@pytest.mark.parametrize("dtype", sorted(NATIVE_SUMS))
def test_integer_and_f64_sums_use_native_red_and_atom(native_lib, dtype):
    (dt, op), add = NATIVE_SUMS[dtype]
    sass = _run("-sass", "-fun", _name(dt, op))
    assert "arch = sm_90a" in sass, sass[:400]
    ops = set(re.findall(r"\b([A-Z][A-Z0-9_]*(?:\.[A-Z0-9_]+)*)\b", sass))
    # plain items reduce, fetching items take the old value back
    assert f"REDG.E.{add}" in ops and f"ATOMG.E.{add}" in ops, sorted(o for o in ops if o.startswith(("RED", "ATOM")))
    assert not any(o.startswith("ATOMG.E.CAS") for o in ops), "a CAS loop where the ISA has the add"
    assert not any(o.startswith(("LDL", "STL")) for o in ops), "local-memory traffic"


def test_no_instantiation_spills(native_lib):
    usage = _run("-res-usage")
    found = re.findall(re.escape(PREFIX) + r"\w+:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", usage)
    # every (dtype, op) of rmaSupported(dtype, op, true): 136 pairs
    assert len(found) == 136, len(found)
    for reg, stack, _, local in found:
        assert int(reg) <= 255 and int(stack) == 0 and int(local) == 0, (reg, stack, local)
