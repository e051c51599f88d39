"""Cost of request-based accumulates (MPI_Raccumulate / MPI_Rget_accumulate,
batched into one accumulate kernel per burst) against plain ones
(MPI_Accumulate / MPI_Get_accumulate, one launch per call).

Runs the `bench-rma-raccumulate` function of faabric_worker: rank 0 applies K
int64 SUM operations from device memory to rank 1's symmetric-heap window
inside MPI_Win_lock_all, as
  * MPI_Raccumulate x K + MPI_Waitall + MPI_Win_flush ("updates": +1 to K
    distinct counters), or MPI_Rget_accumulate x K ("tickets": fetching +1 of
    one counter, a chain that one warp applies in issue order), against
  * MPI_Accumulate / MPI_Get_accumulate x K + MPI_Win_flush,
for K in {1, 64, 1024}, in two layouts:
  * one worker process, two ranks sharing cuda:0 (target in this process:
    the batched path);
  * two worker processes, one rank each (target in another process: both
    calls are shipped at the flush).
It reports µs per operation for every round; the rounds alternate the two
calls.  The card's name and power limit are read in the same call.

    python scripts/bench_mpi_raccumulate.py [--rounds 2] [--json out.json]
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
PATTERNS = ["updates", "tickets"]
MODES = ["racc", "acc"]


def iterations(k, layout):
    # about 4096 operations per case; a tenth of that for the shipped layout
    it = max(3, 4096 // k)
    return max(3, it // 10) if layout[0] > 1 else it


def card():
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


def one_round(tmp: Path, alternate: bool) -> list[dict]:
    rows = []
    for layout in LAYOUTS:
        workers, slots = layout
        with LocalCluster(n_workers=workers, slots_per_worker=slots, log_level="warn", log_dir=tmp) as c:
            for pattern in PATTERNS:
                for k in KS:
                    for mode in (MODES if alternate else MODES[::-1]):
                        payload = f"{mode};{pattern};{k};{iterations(k, layout)}"
                        st = c.client.invoke("mpi", "bench-rma-raccumulate", mpi_world_size=2, input_data=payload, timeout=900)
                        res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
                        if any(m.get("returnValue", 0) != 0 for m in res):
                            raise RuntimeError(f"bench-rma-raccumulate {payload} failed: {res}")
                        target = "this process" if workers == 1 else "other process"
                        rows.append(dict(target=target, mode=mode, pattern=pattern, k=k, **json.loads(res[0]["output_data"])))
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", type=str, default=None)
    a = ap.parse_args()
    print(f"# {card()}")
    rounds = []
    with tempfile.TemporaryDirectory() as d:
        for i in range(a.rounds):
            rounds.append(one_round(Path(d), i % 2 == 0))
    print("| target | pattern | K | request µs/op (rounds) | plain µs/op (rounds) |")
    print("|---|---|---|---|---|")

    def us(rows, key, mode):
        return next(r["us_per_op"] for r in rows if (r["target"], r["pattern"], r["k"]) == key and r["mode"] == mode)

    for r in rounds[0]:
        if r["mode"] != "racc":
            continue
        key = (r["target"], r["pattern"], r["k"])
        rus = " / ".join(f"{us(rr, key, 'racc'):.2f}" for rr in rounds)
        pus = " / ".join(f"{us(rr, key, 'acc'):.2f}" for rr in rounds)
        print(f"| {key[0]} | {key[1]} | {key[2]} | {rus} | {pus} |")
    if a.json:
        Path(a.json).write_text(json.dumps(dict(card=card(), rounds=rounds), indent=1))


if __name__ == "__main__":
    main()
