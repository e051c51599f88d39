"""Throughput and latency of the one-sided accumulate kernel on one GPU.

Ranks share the GPU (LocalGroup); "peer" memory is reached through the same
peer mapping a multi-GPU run uses, but stays in this GPU's HBM, so the
numbers measure the system-scope atomics themselves, not NVLink.

For i32, f32, f16 and f64 SUM at 8 B, 4 KiB, 1 MiB and 64 MiB it times, with
CUDA events over many launches after a warm-up:
  * one writer: rank 0 accumulates into rank 1's window;
  * all writers: every rank accumulates into rank 0's window at once;
  * put: rank 0's put_signal of the same bytes into rank 1's window.
GB/s counts the origin bytes every writer sends.  The card's name and power
limit are read in the same run and printed next to the table.

    python scripts/bench_rma.py [--ranks 4] [--json out.json]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from faabric_b200.parallel import LocalGroup  # noqa: E402

DTYPES = {"i32": torch.int32, "f32": torch.float32, "f16": torch.float16, "f64": torch.float64}
SIZES = [8, 4 << 10, 1 << 20, 64 << 20]
WARMUP = 5


def iters_for(nbytes):
    return 1000 if nbytes <= 4096 else (200 if nbytes <= (1 << 20) else 10)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(
            ["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
            capture_output=True,
            text=True,
            timeout=30,
        )
        limit = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def timed(g, writers, issue, iters):
    """ms from a common start to the last writer's end, for `iters` calls per writer."""
    dev_stream = torch.cuda.current_stream(0)
    start = torch.cuda.Event(enable_timing=True)
    start.record(dev_stream)
    ends = []
    for r in writers:
        st = g.streams[r]
        st.wait_event(start)
        with torch.cuda.stream(st):
            for _ in range(iters):
                issue(r, st)
        e = torch.cuda.Event(enable_timing=True)
        e.record(st)
        ends.append(e)
    torch.cuda.synchronize()
    return max(start.elapsed_time(e) for e in ends)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--ranks", type=int, default=4)
    ap.add_argument("--json", type=str, default=None, help="also write the rows here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rma needs a GPU")
    n = a.ranks
    maxb = max(SIZES)
    g = LocalGroup(n, devices=[0] * n, heapBytes=maxb + (8 << 20), stageBytes=1 << 20, maxBlocks=8, timeoutMs=10000)
    wins = [c.empty(maxb, torch.uint8) for c in g.comms]
    srcs = [torch.empty(maxb, dtype=torch.uint8, device="cuda:0") for _ in range(n)]
    name, limit = card()
    rows = []
    for dname, tdt in DTYPES.items():
        # +1 from even ranks, -1 from odd ones: the targets stay small, so every
        # f16 add still changes the value (an add that changes nothing skips
        # its write on the CAS paths and would time faster than real work)
        for r, s in enumerate(srcs):
            s.view(tdt).fill_(1 if r % 2 == 0 else -1)
        for nbytes in SIZES:
            it = iters_for(nbytes)

            def acc_to(peer):
                return lambda r, st: g.comms[r].accumulate(srcs[r][:nbytes], wins[r][:nbytes], peer, dtype=dname, stream=st)

            modes = {
                "one writer": ([0], acc_to(1)),
                f"{n} writers": (list(range(n)), acc_to(0)),
                "put": ([0], lambda r, st: g.comms[r].put_signal(srcs[r][:nbytes], wins[r][:nbytes], 1, signal=0, blocks=16, stream=st)),
            }
            for mode, (writers, issue) in modes.items():
                for w in wins:
                    w.zero_()
                timed(g, writers, issue, WARMUP)
                ms = timed(g, writers, issue, it)
                us_per_call = ms * 1e3 / it
                gbs = len(writers) * it * nbytes / (ms * 1e-3) / 1e9
                rows.append(dict(dtype=dname, bytes=nbytes, mode=mode, us_per_call=us_per_call, gb_per_s=gbs, iters=it))
    assert g.check_errors() == [0] * n
    g.close()
    print(f"# {name}, power limit / max SM clock: {limit}; {n} ranks sharing cuda:0; SUM")
    print(f"| dtype | bytes | mode | µs per call | GB/s |")
    print("|---|---:|---|---:|---:|")
    for r in rows:
        print(f"| {r['dtype']} | {r['bytes']} | {r['mode']} | {r['us_per_call']:.2f} | {r['gb_per_s']:.3f} |")
    if a.json:
        Path(a.json).write_text(json.dumps(dict(card=name, power_limit=limit, ranks=n, rows=rows), indent=1))


if __name__ == "__main__":
    main()
