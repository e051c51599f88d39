"""MPI_Allreduce on sub-communicators: fused kernels against the host path.

Runs the `bench-subcomm` function of faabric_worker (float32 SUM on
symmetric-heap buffers) in one worker process, all ranks sharing cuda:0:
  * fused: a half communicator (4 ranks) of an 8-rank world, on a signal slot
           (both halves call at the same time);
  * host:  the same call after FB_SUB_SLOTS world splits have taken every slot,
           which is the point-to-point path every sub-communicator took before
           the fused one existed (the device-collective count confirms it);
  * world: MPI_COMM_WORLD of a 4-rank world, which the fused numbers should
           match.
It reports µs per call for every round.  The card's name and power limit are
read in the same call.

    python scripts/bench_subcomm.py [--rounds 2] [--json out.json]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from faabric_b200.runtime import LocalCluster  # noqa: E402

SIZES = [4 << 10, 256 << 10, 4 << 20, 64 << 20]
# (mode, world size); iterations per size come from iters()
MODES = [("fused", 8), ("host", 8), ("world", 4)]


def iters(mode: str, nbytes: int) -> int:
    if mode == "host":
        return 50 if nbytes <= (256 << 10) else (10 if nbytes <= (4 << 20) else 3)
    return 100 if nbytes <= (4 << 20) else 20


def card():
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


# two 64 MiB buffers and the MPI staging arena fit in 512 MiB of heap per rank
HEAP_ENV = {"FAABRIC_SYMM_HEAP_BYTES": str(512 << 20)}


def one_round(tmp: Path) -> dict:
    out = {}
    for mode, world in MODES:
        # a fresh worker per mode: every world wires its own heaps
        with LocalCluster(n_workers=1, slots_per_worker=8, log_level="warn", log_dir=tmp, extra_env=HEAP_ENV) as c:
            for nbytes in SIZES:
                payload = f"{mode};{nbytes};{iters(mode, nbytes)}"
                st = c.client.invoke("mpi", "bench-subcomm", mpi_world_size=world, input_data=payload, timeout=900)
                res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
                if len(res) != world or any(m.get("returnValue", 0) != 0 for m in res):
                    raise RuntimeError(f"bench-subcomm {payload} failed: {res}")
                r = json.loads(res[0]["output_data"])
                # one device call per rank and call: both halves of the 8-rank
                # world call at once; the host path makes none
                want = {"fused": 8, "host": 0, "world": 4}[mode]
                if r["device_calls"] != want:
                    raise RuntimeError(f"bench-subcomm {payload}: {r['device_calls']} device calls per call, expected {want}")
                out[f"{mode}/{nbytes}"] = r["us_per_call"]
                print(f"{mode} {label(nbytes)}: {r['us_per_call']:.1f} us", file=sys.stderr, flush=True)
    return out


def label(nbytes: int) -> str:
    return f"{nbytes >> 20} MiB" if nbytes >= (1 << 20) else f"{nbytes >> 10} KiB"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", type=str, default=None)
    a = ap.parse_args()
    print(f"# {card()}")
    rounds = []
    with tempfile.TemporaryDirectory() as d:
        for _ in range(a.rounds):
            rounds.append(one_round(Path(d)))
    print("| bytes | fused, half of 8 ranks (µs) | host path, half of 8 ranks (µs) | MPI_COMM_WORLD of 4 ranks (µs) |")
    print("|---|---|---|---|")
    for nbytes in SIZES:
        cells = [" / ".join(f"{r[f'{m}/{nbytes}']:.1f}" for r in rounds) for m, _ in MODES]
        print(f"| {label(nbytes)} | " + " | ".join(cells) + " |")
    if a.json:
        Path(a.json).write_text(json.dumps(dict(card=card(), rounds=rounds), indent=1))


if __name__ == "__main__":
    main()
