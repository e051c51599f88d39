"""Cost of the MPI one-sided atomics next to the primitive they launch.

Runs the `bench-rma` function of faabric_worker in a LocalCluster of one
worker process with two ranks sharing cuda:0 (rank 0 onto rank 1's window,
every call followed by its closing MPI_Win_fence):
  * µs per MPI_Fetch_and_op (int64 SUM, symmetric-heap window), with device
    and with host origin / result buffers;
  * GB/s of MPI_Accumulate SUM i32 and f32 at 1 MiB and 64 MiB on heap and
    cudaMalloc windows.
Each round also runs scripts/bench_rma.py (Communicator::accumulate timed with
CUDA events, no fence), so the two alternate; the card's name and power limit
are read in the same call.

    python scripts/bench_mpi_rma.py [--rounds 2] [--json out.json]
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

MIB = 1 << 20
CASES = [("fop", "i64", 8, 2000, "heap", "device"), ("fop", "i64", 8, 2000, "heap", "host")] + [
    ("acc", dt, size, 200 if size == MIB else 20, win, "device")
    for dt in ("i32", "f32")
    for size in (MIB, 64 * MIB)
    for win in ("heap", "cuda")
]


def card():
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


def mpi_round(tmp: Path) -> list[dict]:
    rows = []
    with LocalCluster(n_workers=1, slots_per_worker=2, log_level="warn", log_dir=tmp) as c:
        for kind, dt, size, iters, win, bufs in CASES:
            payload = f"{kind};{dt};{size};{iters};{win};{bufs}"
            st = c.client.invoke("mpi", "bench-rma", mpi_world_size=2, input_data=payload, timeout=600)
            res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
            if any(m.get("returnValue", 0) != 0 for m in res):
                raise RuntimeError(f"bench-rma {payload} failed: {res}")
            out = json.loads(res[0]["output_data"])
            rows.append(dict(call=kind, dtype=dt, bytes=size, window=win, buffers=bufs, **out))
    return rows


def primitive_round(tmp: Path) -> list[dict]:
    out = tmp / "bench_rma.json"
    subprocess.run([sys.executable, str(ROOT / "scripts" / "bench_rma.py"), "--ranks", "2", "--json", str(out)], check=True)
    return json.loads(out.read_text())["rows"]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", type=str, default=None)
    a = ap.parse_args()
    print(f"# {card()}")
    mpi, prim = [], []
    with tempfile.TemporaryDirectory() as d:
        for i in range(a.rounds):
            mpi.append(mpi_round(Path(d)))
            prim.append(primitive_round(Path(d)))
    print("| call | dtype | bytes | window | buffers | µs per call (rounds) | GB/s (rounds) |")
    print("|---|---|---:|---|---|---|---|")
    for k, row in enumerate(mpi[0]):
        us = " / ".join(f"{r[k]['us_per_call']:.1f}" for r in mpi)
        gb = " / ".join(f"{r[k]['gb_per_s']:.1f}" for r in mpi)
        print(f"| {row['call']} | {row['dtype']} | {row['bytes']} | {row['window']} | {row['buffers']} | {us} | {gb} |")
    print("\nCommunicator::accumulate (scripts/bench_rma.py, one writer, SUM):")
    print("| dtype | bytes | µs per call (rounds) | GB/s (rounds) |")
    print("|---|---:|---|---|")
    for k, row in enumerate(prim[0]):
        if row["mode"] != "one writer" or row["dtype"] not in ("i32", "f32") or row["bytes"] < MIB:
            continue
        us = " / ".join(f"{r[k]['us_per_call']:.1f}" for r in prim)
        gb = " / ".join(f"{r[k]['gb_per_s']:.1f}" for r in prim)
        print(f"| {row['dtype']} | {row['bytes']} | {us} | {gb} |")
    if a.json:
        Path(a.json).write_text(json.dumps(dict(card=card(), mpi=mpi, primitive=prim), indent=1))


if __name__ == "__main__":
    main()
