"""Cost of batched one-sided atomics (Communicator.accumulate_many, one
rmaAccumulateManyKernel launch per burst) against one accumulate launch per
update (Communicator.accumulate).

Two ranks share cuda:0 in one process; rank 0 updates rank 1's window, K in
{1, 64, 1024}:
  * "updates": K int64 SUM updates of K distinct counters (free items, spread
    over the grid);
  * "tickets": K fetching int64 increments of ONE counter (one chain: a
    single warp applies them in list order, each waiting for the last).
Two numbers per case, in µs per update:
  * "device": CUDA events around the launches of one burst, with the stream
    held by a sleep kernel until the host has issued the whole burst, so it
    is the GPU's time for the burst and not the host's issue time;
  * "host": wall time from the first issue to the end of a stream
    synchronise, over enough repetitions for about 50 ms (what a Python
    caller waits, argument checks included).
Rounds alternate the batched and the per-update path.  The card's name and
power limit are read in the same call.

    python scripts/bench_rma_accumulate_many.py [--rounds 2] [--json out.json]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from faabric_b200.parallel import LocalGroup  # noqa: E402

KS = [1, 64, 1024]
PATTERNS = ["updates", "tickets"]
MODES = ["many", "single"]


def card():
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


def case(g, pattern, k, mode):
    c = g.comms[0]
    st = g.streams[0]
    win = g.win
    one = torch.ones(1, dtype=torch.int64, device="cuda:0")
    fetch = torch.zeros(k, dtype=torch.int64, device="cuda:0")
    if pattern == "updates":
        dsts = [win[i : i + 1] for i in range(k)]
        fetches = None
    else:
        dsts = [win[:1]] * k
        fetches = list(fetch.split(1))

    def issue():
        if mode == "many":
            c.accumulate_many([one] * k, dsts, [1] * k, fetches=fetches, stream=st)
        else:
            for i in range(k):
                c.accumulate(one, dsts[i], 1, fetch=None if fetches is None else fetches[i], stream=st)

    issue()  # warm-up: module load, staging slots
    st.synchronize()
    # device time: the sleep holds the stream until the burst is issued
    t0 = time.perf_counter()
    issue()
    st.synchronize()
    hold = int(2e9 * (time.perf_counter() - t0)) + 10_000_000  # cycles at ~2 GHz, with margin
    ev0 = torch.cuda.Event(enable_timing=True)
    ev1 = torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(st):
        torch.cuda._sleep(hold)
        ev0.record(st)
        issue()
        ev1.record(st)
    st.synchronize()
    device_us = ev0.elapsed_time(ev1) * 1e3 / k
    reps = 3
    while True:
        t0 = time.perf_counter()
        for _ in range(reps):
            issue()
        st.synchronize()
        dt = time.perf_counter() - t0
        if dt > 0.05 or reps >= 1 << 14:
            break
        reps *= 4
    assert g.check_errors() == [0, 0]
    return device_us, dt / (reps * k) * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    g = LocalGroup(2, devices=[0, 0], heapBytes=64 << 20, stageBytes=1 << 20, maxBlocks=4, timeoutMs=8000)
    try:
        g.win = g.comms[0].empty(1 << 16, torch.int64)
        for c in g.comms[1:]:
            c.empty(1 << 16, torch.int64)
        rows = []
        for rnd in range(args.rounds):
            for pattern in PATTERNS:
                for k in KS:
                    for mode in MODES if rnd % 2 == 0 else MODES[::-1]:
                        dev, host = case(g, pattern, k, mode)
                        rows.append(dict(round=rnd, pattern=pattern, k=k, mode=mode, device_us=round(dev, 3), host_us=round(host, 3)))
                        print(json.dumps(rows[-1]), flush=True)
        out = dict(card=card(), rows=rows)
        print(json.dumps(dict(card=out["card"])))
        if args.json:
            Path(args.json).parent.mkdir(parents=True, exist_ok=True)
            Path(args.json).write_text(json.dumps(out, indent=1))
    finally:
        g.close()


if __name__ == "__main__":
    main()
