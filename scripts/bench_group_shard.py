"""Grouped reduce-scatter and all-gather of the ResNet-50 gradients, against a
per-tensor loop and the grouped all-reduce of the same tensors.

N ranks share cuda:0 in this process (LocalGroup).  Each of the 214 ResNet-50
gradient tensors is split into N shards, padded to a multiple of 16 bytes; all
tensors live in the symmetric heap.  Per step it times, with CUDA events after
warm-up:
  * rs_group / ag_group: one grouped launch for the whole list
    (reduce_scatter_group / all_gather_group with a prepared plan);
  * rs_loop / ag_loop:   one reduce_scatter / all_gather call per tensor;
  * ar_group:            the grouped all-reduce of the full tensors, the
                         reference point (reduce-scatter + all-gather is
                         what sharded data parallelism pays instead).
Every mode is repeated --reps times to show the spread.  The card's name and
power limit are read in the same call.

    python scripts/bench_group_shard.py [--ranks 2] [--steps 20] [--warmup 5] [--reps 5] [--json out.json]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from faabric_b200.models.resnet50_grads import resnet50_grad_sizes  # noqa: E402
from faabric_b200.parallel import LocalGroup  # noqa: E402

MODES = ["rs_group", "ag_group", "rs_loop", "ag_loop", "ar_group"]


def card() -> str:
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


class Setup:
    """Symmetric buffers and plans of one rank for one dtype."""

    def __init__(self, c, n, dtype):
        esize = torch.empty((), dtype=dtype).element_size()
        per_vec = 16 // esize
        # per-rank elements: ceil(size / n), padded to whole 16-byte vectors
        self.shards = [(-(-s // n) + per_vec - 1) // per_vec * per_vec for s in resnet50_grad_sizes()]
        total = sum(self.shards)
        self.full = c.empty(total * n, dtype)  # reduce-scatter input, all-reduce buffer
        self.part = c.empty(total, dtype)  # reduce-scatter output, all-gather input
        self.gath = c.empty(total * n, dtype)  # all-gather output
        self.full.copy_(torch.arange(total * n, device=self.full.device) % 7)
        self.full_v, self.part_v, self.gath_v = [], [], []
        o = 0
        for s in self.shards:
            self.full_v.append(self.full[o * n : (o + s) * n])
            self.gath_v.append(self.gath[o * n : (o + s) * n])
            self.part_v.append(self.part[o : o + s])
            o += s
        self.rs_plan = c.prepare_reduce_scatter_group(self.full_v, self.part_v)
        self.ag_plan = c.prepare_all_gather_group(self.part_v, self.gath_v)
        self.ar_plan = c.prepare_group(self.full_v)
        self.bytes = total * n * esize  # bytes of the full tensors


def step_fn(mode, s):
    """One step of `mode` on every rank's stream.  The per-tensor loops issue
    tensor i on every rank before tensor i+1: ranks sharing a GPU meet at
    stream-ordered barriers, so one rank's stream must never run far ahead
    of calls the host has not yet issued for its peers."""

    def step(g):
        if mode.endswith("_group"):
            plan = {"rs_group": "rs_plan", "ag_group": "ag_plan", "ar_group": "ar_plan"}[mode]
            call = {"rs_group": "reduce_scatter_group", "ag_group": "all_gather_group", "ar_group": "all_reduce_group"}[mode]
            g.run(lambda c, r, st: getattr(c, call)(getattr(s[r], plan)))
            return
        cur = torch.cuda.current_stream()
        for st in g.streams:
            st.wait_stream(cur)
        for i in range(len(s[0].shards)):
            for r, c in enumerate(g.comms):
                with torch.cuda.stream(g.streams[r]):
                    if mode == "rs_loop":
                        c.reduce_scatter(s[r].full_v[i], s[r].part_v[i], stream=g.streams[r])
                    else:
                        c.all_gather(s[r].part_v[i], s[r].gath_v[i], stream=g.streams[r])

    return step


def time_mode(g, fn, steps, warmup) -> float:
    """ms per step: CUDA events on the device's current stream, which every
    rank stream waits for at the start (LocalGroup.run) and joins at the end."""
    cur = torch.cuda.current_stream()
    for _ in range(warmup):
        fn(g)
    torch.cuda.synchronize()
    start = torch.cuda.Event(enable_timing=True)
    end = torch.cuda.Event(enable_timing=True)
    start.record(cur)
    for _ in range(steps):
        fn(g)
    for st in g.streams:
        cur.wait_stream(st)
    end.record(cur)
    end.synchronize()
    if g.check_errors() != [0] * g.size:
        raise RuntimeError("device watchdog fired")
    return start.elapsed_time(end) / steps


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--ranks", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    the_card = card()
    print(f"# {the_card}; {a.ranks} ranks on cuda:0", flush=True)
    g = LocalGroup(a.ranks, devices=[0] * a.ranks, heapBytes=320 << 20, stageBytes=8 << 20, timeoutMs=20000)
    results = {}
    try:
        for dtype, name in ((torch.float32, "fp32"), (torch.bfloat16, "bf16")):
            s = [Setup(c, a.ranks, dtype) for c in g.comms]
            for mode in MODES:
                ms = [time_mode(g, step_fn(mode, s), a.steps, a.warmup) for _ in range(a.reps)]
                results[f"{name}/{mode}"] = ms
                print(json.dumps(dict(dtype=name, mode=mode, ms_per_step=[round(x, 4) for x in ms], mib=round(s[0].bytes / 2**20, 1))), flush=True)
            for x in s:
                x.rs_plan.close()
                x.ag_plan.close()
                x.ar_plan.close()
            for c, x in zip(g.comms, s):
                c.free(x.full)
                c.free(x.part)
                c.free(x.gath)
    finally:
        g.close()
    print()
    print(f"ms per step, {a.reps} repetitions of {a.steps} steps (min / median / max), {the_card}")
    print("| dtype | " + " | ".join(MODES) + " |")
    print("|---|" + "---|" * len(MODES))
    for name in ("fp32", "bf16"):
        cells = []
        for mode in MODES:
            v = sorted(results[f"{name}/{mode}"])
            cells.append(f"{v[0]:.3f} / {v[len(v) // 2]:.3f} / {v[-1]:.3f}")
        print(f"| {name} | " + " | ".join(cells) + " |")
    if a.json:
        Path(a.json).write_text(json.dumps(dict(card=the_card, ranks=a.ranks, results=results), indent=1))


if __name__ == "__main__":
    main()
