"""Cost of MPI passive-target synchronisation.

Runs the `bench-rma-passive` function of faabric_worker (rank 0 onto rank 1's
window) in two layouts:
  * one worker process, two ranks sharing cuda:0 (target in this process);
  * two worker processes, one rank each (target in another process: lock,
    flush and unlock go to its point-to-point server).
It reports µs per MPI_Fetch_and_op + MPI_Win_flush inside MPI_Win_lock_all,
the same call closed by MPI_Win_fence instead, and one MPI_Win_lock +
MPI_Win_unlock round trip.  The card's name and power limit are read in the
same call.

    python scripts/bench_mpi_passive.py [--rounds 2] [--json out.json]
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

# (layout, mode, window, buffers, iterations); layout = (workers, ranks per worker)
CASES = [
    ((1, 2), "flush", "heap", "device", 2000),
    ((1, 2), "fence", "heap", "device", 2000),
    ((1, 2), "flush", "host", "host", 2000),
    ((1, 2), "lock", "heap", "device", 2000),
    ((2, 1), "flush", "heap", "device", 500),
    ((2, 1), "fence", "heap", "device", 500),
    ((2, 1), "flush", "host", "host", 500),
    ((2, 1), "lock", "host", "host", 500),
]


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
    for layout in sorted({c[0] for c in CASES}):
        workers, slots = layout
        with LocalCluster(n_workers=workers, slots_per_worker=slots, log_level="warn", log_dir=tmp) as c:
            for lay, mode, win, bufs, iters in CASES:
                if lay != layout:
                    continue
                payload = f"{mode};{win};{bufs};{iters}"
                st = c.client.invoke("mpi", "bench-rma-passive", mpi_world_size=2, input_data=payload, timeout=600)
                res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
                if any(m.get("returnValue", 0) != 0 for m in res):
                    raise RuntimeError(f"bench-rma-passive {payload} failed: {res}")
                target = "this process" if workers == 1 else "other process"
                rows.append(dict(target=target, mode=mode, window=win, buffers=bufs, **json.loads(res[0]["output_data"])))
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
    print("| target | call | window | buffers | µs per call (rounds) |")
    print("|---|---|---|---|---|")
    names = {"flush": "Fetch_and_op + Win_flush", "fence": "Fetch_and_op + Win_fence", "lock": "Win_lock + Win_unlock"}
    for k, row in enumerate(rounds[0]):
        us = " / ".join(f"{r[k]['us_per_call']:.1f}" for r in rounds)
        print(f"| {row['target']} | {names[row['mode']]} | {row['window']} | {row['buffers']} | {us} |")
    if a.json:
        Path(a.json).write_text(json.dumps(dict(card=card(), rounds=rounds), indent=1))


if __name__ == "__main__":
    main()
