"""Cost of request-based puts (MPI_Rput, batched into one copy kernel per
burst) against plain MPI_Put (one synchronous copy per call).

Runs the `bench-rma-request` function of faabric_worker: rank 0 writes K
operations of B bytes from device memory into rank 1's symmetric-heap window
inside MPI_Win_lock_all, as
  * MPI_Rput x K + MPI_Waitall + MPI_Win_flush, and
  * MPI_Put x K + MPI_Win_flush,
for K in {1, 64, 1024} and B in {8 B, 256 B, 64 KiB}, in two layouts:
  * one worker process, two ranks sharing cuda:0 (target in this process:
    the batched path);
  * two worker processes, one rank each (target in another process: both
    calls are shipped at the flush).
It reports µs per operation for every round.  The card's name and power
limit are read in the same call.

    python scripts/bench_mpi_rput.py [--rounds 2] [--json out.json]
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

LAYOUTS = [(1, 2), (2, 1)]  # (workers, ranks per worker)
KS = [1, 64, 1024]
SIZES = [8, 256, 64 << 10]
MODES = ["rput", "put"]


def iterations(k, size, layout):
    # about the same bytes per case; fewer for the shipped layout
    it = max(3, min(2000, (4 << 20) // (k * size)))
    return max(3, it // 10) if layout[0] > 1 else it


def card():
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


def one_round(tmp: Path) -> list[dict]:
    rows = []
    for layout in LAYOUTS:
        workers, slots = layout
        with LocalCluster(n_workers=workers, slots_per_worker=slots, log_level="warn", log_dir=tmp) as c:
            for size in SIZES:
                for k in KS:
                    for mode in MODES:
                        payload = f"{mode};{size};{k};{iterations(k, size, layout)}"
                        st = c.client.invoke("mpi", "bench-rma-request", mpi_world_size=2, input_data=payload, timeout=900)
                        res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
                        if any(m.get("returnValue", 0) != 0 for m in res):
                            raise RuntimeError(f"bench-rma-request {payload} failed: {res}")
                        target = "this process" if workers == 1 else "other process"
                        rows.append(dict(target=target, mode=mode, bytes=size, k=k, **json.loads(res[0]["output_data"])))
    return rows


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
    print("| target | bytes | K | MPI_Rput µs/op (rounds) | MPI_Put µs/op (rounds) |")
    print("|---|---|---|---|---|")
    first = rounds[0]
    for i in range(0, len(first), 2):
        r, p = first[i], first[i + 1]
        rus = " / ".join(f"{rr[i]['us_per_op']:.2f}" for rr in rounds)
        pus = " / ".join(f"{rr[i + 1]['us_per_op']:.2f}" for rr in rounds)
        assert r["mode"] == "rput" and p["mode"] == "put"
        print(f"| {r['target']} | {r['bytes']} | {r['k']} | {rus} | {pus} |")
    if a.json:
        Path(a.json).write_text(json.dumps(dict(card=card(), rounds=rounds), indent=1))


if __name__ == "__main__":
    main()
