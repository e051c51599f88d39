"""Grouped scan and exscan against one prefix-reduction call per tensor,
ranks sharing cuda:0 at 2, 4 and 8 ranks, on two lists that sit on either
side of the grouping trade-off:

  (a) moe: 64 int64 per-expert token-count tensors of 256 experts each on
      every rank, exclusive sum (each rank's write offsets into every
      expert's buffer, once per MoE layer): many tiny items, where launches
      and barriers dominate;
  (b) large: three 32 MiB fp32 tensors on every rank, inclusive sum: few
      large items, where bandwidth dominates and staging costs the most.

Arms, each as one call per tensor against the grouped call:
  * device layer, on a LocalGroup: a per-tensor loop (loop: the blocking
    `scan`; for the exscan, which has no blocking device call, a one-item
    `scan_many`) against one `scan_many` of the list (many), and against one
    `scan_group` launch of a plan prepared once (plan).  ms per step from CUDA
    events (min / median / max over repetitions), device launches per step per
    rank (the communicators' stats), and host µs per call (wall time to issue
    one step, divided by the calls it replaces);
  * MPI, through the `bench-group-scan` function of faabric_worker on one
    worker process whose ranks share cuda:0: k x MPI_Exscan against k x
    MPI_Iexscan + MPI_Waitall (moe), k x MPI_Scan against k x MPI_Iscan +
    MPI_Waitall (large); wall-clock ms per step on rank 0, µs per call = ms
    per step / k, rank 0's launches per step, and the part of a step spent in
    MPI_Waitall.  Every invocation is bounded at 180 s; the MPI arms run at
    MPI_RANKS (see there).
The HBM lower bound of one step is 2 * N * S / 3.35 TB/s (H100 SXM data-sheet
bandwidth, S one rank's bytes: every rank's input is read and its output
written at least once); its fraction of the median is reported, not a
target.  The card's name and power limit are read in the same run.

    python scripts/bench_group_scan.py [--steps 10] [--warmup 3] [--reps 3] [--json out.json] [--no-mpi]
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

from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.runtime import LocalCluster  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
RANKS = (2, 4, 8)
# As the other rooted benchmarks: the MPI arms run at 2 ranks by default, and
# no invocation may hold the GPU for long (docs/next_steps.md).
MPI_RANKS = (2,)
INVOKE_TIMEOUT_S = 180
# name: (elements per tensor, torch dtype, FbDtype name, exclusive)
WORKLOADS = {
    "moe": ([256] * 64, torch.int64, "i64", True),
    "large": ([(32 << 20) // 4] * 3, torch.float32, "f32", False),
}


def card() -> str:
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


def tensors(c, counts, dtype):
    """One rank's send and recv views of each tensor, in two heap buffers"""
    total = sum(counts)
    send = c.empty(total, dtype)
    recv = c.empty(total, dtype)
    send.copy_(torch.arange(total, device=send.device) % 251)
    recv.zero_()
    sv, rv, o = [], [], 0
    for k in counts:
        sv.append(send[o : o + k])
        rv.append(recv[o : o + k])
        o += k
    return (send, recv), sv, rv


def loop(g, sends, recvs, exclusive):
    """Tensor i on every rank before tensor i+1"""
    cur = torch.cuda.current_stream()
    for st in g.streams:
        st.wait_stream(cur)
    for i in range(len(sends[0])):
        for r, c in enumerate(g.comms):
            with torch.cuda.stream(g.streams[r]):
                if exclusive:
                    c.scan_many([sends[r][i]], [recvs[r][i]], exclusive=True, stream=g.streams[r])
                else:
                    c.scan(sends[r][i], recvs[r][i], op="sum", stream=g.streams[r])


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
        for name, (counts, dtype, _, ex) in WORKLOADS.items():
            made = [tensors(c, counts, dtype) for c in g.comms]
            sends = [m[1] for m in made]
            recvs = [m[2] for m in made]
            es = torch.empty(0, dtype=dtype).element_size()
            bound_ms = 2 * n * sum(counts) * es / HBM_BYTES_PER_S * 1e3
            plans = [c.prepare_scan_group(sends[r], recvs[r], exclusive=ex) for r, c in enumerate(g.comms)]
            kind = "exscan" if ex else "scan"
            modes = {
                "loop": lambda: loop(g, sends, recvs, ex),
                "many": lambda: g.run(lambda c, r, st: c.scan_many(sends[r], recvs[r], exclusive=ex)),
                "plan": lambda: g.run(lambda c, r, st: c.scan_group(plans[r])),
            }
            for mode, fn in modes.items():
                reps = [measure(g, fn, a.steps, a.warmup, len(counts)) for _ in range(a.reps)]
                r = row([x[0] for x in reps], reps[0][1], sorted(x[2] for x in reps)[len(reps) // 2], bound_ms)
                out[f"{name}/{kind}_{mode}"] = r
                mib = round(sum(counts) * es / 2**20, 3)
                print(json.dumps(dict(ranks=n, workload=name, mode=f"{kind}_{mode}", mib_per_rank=mib, **r)), flush=True)
            # the grouped call and the loop leave the same values on every rank
            for rv in recvs:
                for t in rv:
                    t.zero_()
            modes["many"]()
            torch.cuda.synchronize()
            grouped = [torch.cat([t.view(-1) for t in rv]).clone() for rv in recvs]
            modes["loop"]()
            torch.cuda.synchronize()
            for r, rv in enumerate(recvs):
                if not torch.equal(grouped[r], torch.cat([t.view(-1) for t in rv])):
                    raise RuntimeError(f"{name}: grouped and per-tensor results differ on rank {r}")
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
            for name, (counts, dtype, fbd, ex) in WORKLOADS.items():
                es = torch.empty(0, dtype=dtype).element_size()
                bound_ms = 2 * n * sum(counts) * es / HBM_BYTES_PER_S * 1e3
                kind = "exscan" if ex else "scan"
                for mode in (kind, "i" + kind):
                    reps = []
                    for _ in range(a.reps):
                        st = c.client.invoke(
                            "mpi",
                            "bench-group-scan",
                            mpi_world_size=n,
                            input_data=f"{mode};{a.steps};{fbd};{','.join(map(str, counts))}",
                            timeout=INVOKE_TIMEOUT_S,
                        )
                        res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
                        if any(m.get("returnValue", 0) != 0 for m in res):
                            raise RuntimeError(f"bench-group-scan {mode} on {n} ranks failed: {res}")
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
