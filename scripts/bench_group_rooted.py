"""Grouped gather and scatter against one call per tensor, ranks sharing
cuda:0 at 2, 4 and 8 ranks, gathering to and scattering from rank 0, on two
lists that sit on either side of the grouping trade-off:

  (a) resnet50: each rank's 1/N shard of the 214 ResNet-50 tensors (fp32),
      as in saving (gather) or loading (scatter) a full state dict of a
      sharded data-parallel model: many small items, where launches and
      barriers dominate;
  (b) large: three 32 MiB fp32 tensors at the root, 32/N MiB per rank: few
      large items, where bandwidth dominates.

Arms, each as one call per tensor against the grouped call:
  * device layer, on a LocalGroup: a per-tensor `gather` / `scatter` loop
    (loop) against one `gather_many` / `scatter_many` of the list (many), and
    against one `gather_group` / `scatter_group` launch of a plan prepared
    once (plan).  ms per step from CUDA events (min / median / max over
    repetitions), device launches per step per rank (the communicators'
    stats), and host µs per call (wall time to issue one step, divided by the
    calls it replaces);
  * MPI, through the `bench-group-rooted` function of faabric_worker on one
    worker process whose ranks share cuda:0: k x MPI_Gather / MPI_Scatter
    against k x MPI_Igather / MPI_Iscatter + MPI_Waitall, wall-clock ms per
    step on rank 0, µs per call = ms per step / k, rank 0's launches per
    step, and the part of a step spent in MPI_Waitall.  Every invocation is
    bounded at 180 s; the MPI arms run at MPI_RANKS (see there).
The HBM lower bound of one step is 2 * N * S / 3.35 TB/s (H100 SXM data-sheet
bandwidth, S one rank's bytes: the root reads and writes N * S at least); its
fraction of the median is reported, not a target.  The card's name and power
limit are read in the same run.

    python scripts/bench_group_rooted.py [--steps 10] [--warmup 3] [--reps 3] [--json out.json] [--no-mpi]
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
# 214 blocking MPI_Scatter calls at 4 ranks sharing one GPU once stopped
# making progress in this benchmark, after the MPI_Igather arm in the same
# worker process (docs/next_steps.md); until that is understood the MPI arms
# run at 2 ranks by default, and no invocation may hold the GPU for long.
MPI_RANKS = (2,)
INVOKE_TIMEOUT_S = 180
OPS = ("gather", "scatter")


def card() -> str:
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


def workload(name: str, n: int) -> list[int]:
    """One rank's bytes per tensor"""
    if name == "resnet50":
        return [(s + n - 1) // n * 4 for s in resnet50_grad_sizes()]
    return [(32 << 20) // n] * 3


def tensors(c, sizes, n, root_side):
    """One rank's single-block and n-block views of each tensor (fp32), in two
    heap buffers; the n-block side only where `root_side`"""
    total = sum(sizes) // 4
    one = c.empty(total, torch.float32)
    many = c.empty(total * n, torch.float32)
    one.copy_(torch.arange(total, device=one.device) % 251)
    many.copy_(torch.arange(total * n, device=many.device) % 253)
    ov, mv, o = [], [], 0
    for s in sizes:
        ov.append(one[o : o + s // 4])
        mv.append(many[o * n : (o + s // 4) * n] if root_side else None)
        o += s // 4
    return (one, many), ov, mv


def loop(g, op, ones, manys):
    """Tensor i on every rank before tensor i+1"""
    cur = torch.cuda.current_stream()
    for st in g.streams:
        st.wait_stream(cur)
    for i in range(len(ones[0])):
        for r, c in enumerate(g.comms):
            with torch.cuda.stream(g.streams[r]):
                if op == "gather":
                    c.gather(ones[r][i], manys[r][i], root=0, stream=g.streams[r], flags=0)
                else:
                    c.scatter(manys[r][i], ones[r][i], root=0, stream=g.streams[r], flags=0)


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
            sizes = workload(name, n)
            made = [tensors(c, sizes, n, r == 0) for r, c in enumerate(g.comms)]
            ones = [m[1] for m in made]
            manys = [m[2] for m in made]
            bound_ms = 2 * n * sum(sizes) / HBM_BYTES_PER_S * 1e3
            for op in OPS:
                if op == "gather":
                    plans = [c.prepare_gather_group(ones[r], manys[r] if r == 0 else None) for r, c in enumerate(g.comms)]
                    many = lambda c, r: c.gather_many(ones[r], manys[r] if r == 0 else None)  # noqa: E731
                    grp = lambda c, r: c.gather_group(plans[r])  # noqa: E731
                else:
                    plans = [c.prepare_scatter_group(manys[r] if r == 0 else None, ones[r]) for r, c in enumerate(g.comms)]
                    many = lambda c, r: c.scatter_many(manys[r] if r == 0 else None, ones[r])  # noqa: E731
                    grp = lambda c, r: c.scatter_group(plans[r])  # noqa: E731
                modes = {
                    "loop": lambda: loop(g, op, ones, manys),
                    "many": lambda: g.run(lambda c, r, st: many(c, r)),
                    "plan": lambda: g.run(lambda c, r, st: grp(c, r)),
                }
                for mode, fn in modes.items():
                    reps = [measure(g, fn, a.steps, a.warmup, len(sizes)) for _ in range(a.reps)]
                    r = row([x[0] for x in reps], reps[0][1], sorted(x[2] for x in reps)[len(reps) // 2], bound_ms)
                    out[f"{name}/{op}_{mode}"] = r
                    print(json.dumps(dict(ranks=n, workload=name, mode=f"{op}_{mode}", mib_per_rank=round(sum(sizes) / 2**20, 2), **r)), flush=True)
                # the grouped call and the loop leave the same bytes
                side = [manys[0]] if op == "gather" else ones
                for tv in side:
                    for t in tv:
                        t.zero_()
                modes["many"]()
                torch.cuda.synchronize()
                grouped = [torch.cat([t.view(-1) for t in tv]).clone() for tv in side]
                modes["loop"]()
                torch.cuda.synchronize()
                for r, tv in enumerate(side):
                    if not torch.equal(grouped[r], torch.cat([t.view(-1) for t in tv])):
                        raise RuntimeError(f"{name} {op}: grouped and per-tensor results differ on rank {r}")
                for p in plans:
                    p.close()
            for c, ((o, m), _, _) in zip(g.comms, made):
                c.free(o)
                c.free(m)
    finally:
        g.close()
    return out


def bench_mpi(a, tmp):
    out = {}
    for n in a.mpi_ranks:
        with LocalCluster(n_workers=1, slots_per_worker=n, log_level="warn", log_dir=tmp) as c:
            for name in ("resnet50", "large"):
                sizes = workload(name, n)
                bound_ms = 2 * n * sum(sizes) / HBM_BYTES_PER_S * 1e3
                for mode in ("gather", "igather", "scatter", "iscatter"):
                    reps = []
                    for _ in range(a.reps):
                        st = c.client.invoke(
                            "mpi",
                            "bench-group-rooted",
                            mpi_world_size=n,
                            input_data=f"{mode};{a.steps};{','.join(map(str, sizes))}",
                            timeout=INVOKE_TIMEOUT_S,
                        )
                        res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
                        if any(m.get("returnValue", 0) != 0 for m in res):
                            raise RuntimeError(f"bench-group-rooted {mode} on {n} ranks failed: {res}")
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
