"""Grouped reduce against one MPI_Reduce-style call per tensor, ranks sharing
cuda:0 at 2, 4 and 8 ranks, reducing (sum) to rank 0, on two lists that sit
on either side of the grouping trade-off:

  (a) resnet50: the 214 full ResNet-50 fp32 gradient tensors on every rank,
      as collected by a parameter-server or optimizer rank: many small items,
      where launches and barriers dominate;
  (b) large: three 32 MiB fp32 tensors on every rank: few large items, where
      bandwidth dominates.

Arms, each as one call per tensor against the grouped call:
  * device layer, on a LocalGroup: a per-tensor `reduce` loop (loop) against
    one `reduce_many` of the list (many), and against one `reduce_group`
    launch of a plan prepared once (plan).  ms per step from CUDA events
    (min / median / max over repetitions), device launches per step per rank
    (the communicators' stats), and host µs per call (wall time to issue one
    step, divided by the calls it replaces);
  * MPI, through the `bench-group-reduce` function of faabric_worker on one
    worker process whose ranks share cuda:0: k x MPI_Reduce against k x
    MPI_Ireduce + MPI_Waitall, wall-clock ms per step on rank 0, µs per call
    = ms per step / k, rank 0's launches per step, and the part of a step
    spent in MPI_Waitall.  Every invocation is bounded at 180 s; the MPI arms
    run at MPI_RANKS (see there).
The HBM lower bound of one step is (N + 1) * S / 3.35 TB/s (H100 SXM
data-sheet bandwidth, S one rank's bytes: every rank's input is read and the
root's output written at least once); its fraction of the median is
reported, not a target.  The card's name and power limit are read in the
same run.

    python scripts/bench_group_reduce.py [--steps 10] [--warmup 3] [--reps 3] [--json out.json] [--no-mpi]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from faabric_b200.models.resnet50_grads import resnet50_grad_sizes  # noqa: E402
from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.runtime import LocalCluster  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
RANKS = (2, 4, 8)
# Blocking rooted collectives at 4 ranks sharing one GPU once stopped making
# progress (docs/next_steps.md); until that is understood the MPI arms run at
# 2 ranks by default, and no invocation may hold the GPU for long.
MPI_RANKS = (2,)
INVOKE_TIMEOUT_S = 180


def card() -> str:
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


def workload(name: str) -> list[int]:
    """Elements per tensor (fp32), the same on every rank"""
    if name == "resnet50":
        return resnet50_grad_sizes()
    return [(32 << 20) // 4] * 3


def tensors(c, counts):
    """One rank's send and recv views of each tensor, in two heap buffers"""
    total = sum(counts)
    send = c.empty(total, torch.float32)
    recv = c.empty(total, torch.float32)
    send.copy_(torch.arange(total, device=send.device) % 251)
    recv.zero_()
    sv, rv, o = [], [], 0
    for k in counts:
        sv.append(send[o : o + k])
        rv.append(recv[o : o + k])
        o += k
    return (send, recv), sv, rv


def loop(g, sends, recvs):
    """Tensor i on every rank before tensor i+1"""
    cur = torch.cuda.current_stream()
    for st in g.streams:
        st.wait_stream(cur)
    for i in range(len(sends[0])):
        for r, c in enumerate(g.comms):
            with torch.cuda.stream(g.streams[r]):
                c.reduce(sends[r][i], recvs[r][i], root=0, op="sum", stream=g.streams[r])


def measure(g, fn, steps, warmup, calls):
    """(ms per step, launches per step per rank, host µs per replaced call)"""
    cur = torch.cuda.current_stream()
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    l0 = [c.stats()["launches"] for c in g.comms]
    start = torch.cuda.Event(enable_timing=True)
    end = torch.cuda.Event(enable_timing=True)
    start.record(cur)
    host = 0.0
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        host += time.perf_counter() - t0
    for st in g.streams:
        cur.wait_stream(st)
    end.record(cur)
    end.synchronize()
    if g.check_errors() != [0] * g.size:
        raise RuntimeError("device watchdog fired")
    launches = max(c.stats()["launches"] - b for c, b in zip(g.comms, l0)) / steps
    return start.elapsed_time(end) / steps, launches, host / steps / calls * 1e6


def row(ms: list[float], launches: float, host_us: float, bound_ms: float) -> dict:
    ms = sorted(ms)
    return dict(
        ms_per_step=dict(min=round(ms[0], 4), median=round(ms[len(ms) // 2], 4), max=round(ms[-1], 4)),
        launches_per_step=launches,
        host_us_per_call=round(host_us, 2),
        hbm_bound_fraction=round(bound_ms / ms[len(ms) // 2], 3),
    )


def bench_device(n, a):
    g = LocalGroup(n, devices=[0] * n, heapBytes=512 << 20, timeoutMs=20000)
    out = {}
    try:
        for name in ("resnet50", "large"):
            counts = workload(name)
            made = [tensors(c, counts) for c in g.comms]
            sends = [m[1] for m in made]
            recvs = [m[2] for m in made]
            roots = [recvs[0]] + [None] * (n - 1)
            bound_ms = (n + 1) * sum(counts) * 4 / HBM_BYTES_PER_S * 1e3
            plans = [c.prepare_reduce_group(sends[r], roots[r]) for r, c in enumerate(g.comms)]
            modes = {
                "loop": lambda: loop(g, sends, recvs),
                "many": lambda: g.run(lambda c, r, st: c.reduce_many(sends[r], roots[r])),
                "plan": lambda: g.run(lambda c, r, st: c.reduce_group(plans[r])),
            }
            for mode, fn in modes.items():
                reps = [measure(g, fn, a.steps, a.warmup, len(counts)) for _ in range(a.reps)]
                r = row([x[0] for x in reps], reps[0][1], sorted(x[2] for x in reps)[len(reps) // 2], bound_ms)
                out[f"{name}/reduce_{mode}"] = r
                print(json.dumps(dict(ranks=n, workload=name, mode=f"reduce_{mode}", mib_per_rank=round(sum(counts) * 4 / 2**20, 2), **r)), flush=True)
            # the grouped call and the loop leave the same values at the root
            for t in recvs[0]:
                t.zero_()
            modes["many"]()
            torch.cuda.synchronize()
            grouped = torch.cat([t.view(-1) for t in recvs[0]]).clone()
            modes["loop"]()
            torch.cuda.synchronize()
            if not torch.equal(grouped, torch.cat([t.view(-1) for t in recvs[0]])):
                raise RuntimeError(f"{name}: grouped and per-tensor results differ at the root")
            for p in plans:
                p.close()
            for c, ((s, rv), _, _) in zip(g.comms, made):
                c.free(s)
                c.free(rv)
    finally:
        g.close()
    return out


def bench_mpi(a, tmp):
    out = {}
    for n in a.mpi_ranks:
        with LocalCluster(n_workers=1, slots_per_worker=n, log_level="warn", log_dir=tmp) as c:
            for name in ("resnet50", "large"):
                counts = workload(name)
                bound_ms = (n + 1) * sum(counts) * 4 / HBM_BYTES_PER_S * 1e3
                for mode in ("reduce", "ireduce"):
                    reps = []
                    for _ in range(a.reps):
                        st = c.client.invoke(
                            "mpi",
                            "bench-group-reduce",
                            mpi_world_size=n,
                            input_data=f"{mode};{a.steps};{','.join(map(str, counts))}",
                            timeout=INVOKE_TIMEOUT_S,
                        )
                        res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
                        if any(m.get("returnValue", 0) != 0 for m in res):
                            raise RuntimeError(f"bench-group-reduce {mode} on {n} ranks failed: {res}")
                        reps.append(json.loads(res[0]["output_data"]))
                    r = row(
                        [x["ms_per_step"] for x in reps],
                        reps[0]["launches_per_step"],
                        sorted(x["us_per_call"] for x in reps)[len(reps) // 2],
                        bound_ms,
                    )
                    r["wait_ms_per_step"] = round(sorted(x["wait_ms_per_step"] for x in reps)[len(reps) // 2], 4)
                    out[f"{n}/{name}/{mode}"] = r
                    print(json.dumps(dict(ranks=n, workload=name, mode=f"mpi {mode}", **r)), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", type=str, default=None)
    ap.add_argument("--no-mpi", action="store_true", help="only the device-layer calls")
    ap.add_argument("--no-device", action="store_true", help="only the MPI calls")
    ap.add_argument("--mpi-ranks", type=int, nargs="+", default=list(MPI_RANKS), help="world sizes of the MPI comparison")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    the_card = card()
    print(f"# {the_card}", flush=True)
    results = {}
    if not a.no_device:
        results.update({f"device/{n}": bench_device(n, a) for n in RANKS})
    if not a.no_mpi:
        with tempfile.TemporaryDirectory() as d:
            results["mpi"] = bench_mpi(a, Path(d))
    if a.json:
        Path(a.json).write_text(json.dumps(dict(card=the_card, results=results), indent=1))


if __name__ == "__main__":
    main()
