"""Grouped all-to-all against one call per tensor, ranks sharing cuda:0 at 2,
4 and 8 ranks, on two lists that sit on either side of the grouping trade-off:

  (a) resnet50: the 214 ResNet-50 gradient tensors (fp32), each padded to a
      multiple of 16 * N bytes, as one rank's sends (97.6 MiB): many small
      blocks, where launches and barriers dominate;
  (b) ulysses: three 32 MiB bf16 tensors per rank (Q/K/V of a 4096-token x
      4096-hidden shard in Ulysses sequence parallelism): few large blocks,
      where bandwidth dominates.

Arms, each as one call per tensor against the grouped call:
  * device layer, on a LocalGroup: a per-tensor `all_to_all` loop
    (a2a_loop) against one `all_to_all_many` of the list (a2a_many), and
    against one `all_to_all_group` launch of a plan prepared once
    (a2a_plan: no per-step list marshalling or table upload).  ms per step
    from CUDA events (min / median / max over repetitions), device launches
    per step per rank (the communicators' stats), and host µs per call (wall
    time to issue one step, divided by the calls it replaces);
  * MPI, through the `bench-group-alltoall` function of faabric_worker on one
    worker process whose ranks share cuda:0: k x MPI_Alltoall (mpi alltoall)
    against k x MPI_Ialltoall + MPI_Waitall (mpi ialltoall), wall-clock ms per
    step on rank 0, µs per call = ms per step / k, rank 0's launches per
    step, and the part of a step spent in MPI_Waitall (where a burst is
    issued and completed).  Workload (b) runs through MPI at the ranks of
    MPI_ULYSSES_RANKS only (see there).
The HBM lower bound of one step is 2 * N * S / 3.35 TB/s (H100 SXM data-sheet
bandwidth, S one rank's send bytes: each rank reads S and writes S, and the N
ranks share one card's HBM); its fraction of the median is reported, not a
target.  The card's name and power limit are read in the same run.

    python scripts/bench_group_alltoall.py [--steps 10] [--warmup 3] [--reps 3] [--json out.json] [--no-mpi]
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
# Three blocking MPI_Alltoall calls of 8 MiB blocks at 4 ranks sharing one
# GPU stopped making progress in this benchmark (docs/next_steps.md); until
# that is understood, workload (b) goes through MPI at 2 ranks only, and no
# invocation may hold the GPU for long.
MPI_ULYSSES_RANKS = (2,)
INVOKE_TIMEOUT_S = 180


def card() -> str:
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


def workload(name: str, n: int) -> tuple[list[int], torch.dtype]:
    """One rank's send bytes per tensor (multiples of 16 * n) and the dtype"""
    if name == "resnet50":
        q = 16 * n
        return [(s * 4 + q - 1) // q * q for s in resnet50_grad_sizes()], torch.float32
    return [32 << 20] * 3, torch.bfloat16


def tensors(c, sizes, dtype):
    """Send and recv views of each tensor, in two heap buffers of one rank"""
    es = torch.empty((), dtype=dtype).element_size()
    total = sum(sizes) // es
    send = c.empty(total, dtype)
    recv = c.empty(total, dtype)
    send.copy_((torch.arange(total, device=send.device) % 251).to(dtype))
    recv.zero_()
    sv, rv, o = [], [], 0
    for s in sizes:
        sv.append(send[o : o + s // es])
        rv.append(recv[o : o + s // es])
        o += s // es
    return (send, recv), sv, rv


def loop(g, sends, recvs):
    """Tensor i on every rank before tensor i+1 (stream-ordered barriers
    between ranks sharing a GPU)."""
    cur = torch.cuda.current_stream()
    for st in g.streams:
        st.wait_stream(cur)
    for i in range(len(sends[0])):
        for r, c in enumerate(g.comms):
            with torch.cuda.stream(g.streams[r]):
                c.all_to_all(sends[r][i], recvs[r][i], stream=g.streams[r])


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
    g = LocalGroup(n, devices=[0] * n, heapBytes=512 << 20, stageBytes=8 << 20, timeoutMs=20000)
    out = {}
    try:
        for name in ("resnet50", "ulysses"):
            sizes, dtype = workload(name, n)
            made = [tensors(c, sizes, dtype) for c in g.comms]
            sends = [m[1] for m in made]
            recvs = [m[2] for m in made]
            bound_ms = 2 * n * sum(sizes) / HBM_BYTES_PER_S * 1e3
            plans = [c.prepare_all_to_all_group(sends[r], recvs[r]) for r, c in enumerate(g.comms)]
            modes = {
                "a2a_loop": lambda: loop(g, sends, recvs),
                "a2a_many": lambda: g.run(lambda c, r, st: c.all_to_all_many(sends[r], recvs[r])),
                "a2a_plan": lambda: g.run(lambda c, r, st: c.all_to_all_group(plans[r])),
            }
            for mode, fn in modes.items():
                reps = [measure(g, fn, a.steps, a.warmup, len(sizes)) for _ in range(a.reps)]
                r = row([x[0] for x in reps], reps[0][1], sorted(x[2] for x in reps)[len(reps) // 2], bound_ms)
                out[f"{name}/{mode}"] = r
                print(json.dumps(dict(ranks=n, workload=name, mode=mode, send_mib=round(sum(sizes) / 2**20, 1), **r)), flush=True)
            # the grouped call and the loop leave the same bytes
            fn = modes["a2a_many"]
            for rv in recvs:
                for t in rv:
                    t.zero_()
            fn()
            torch.cuda.synchronize()
            grouped = [torch.cat([t.view(torch.uint8) for t in rv]).clone() for rv in recvs]
            modes["a2a_loop"]()
            torch.cuda.synchronize()
            for r, rv in enumerate(recvs):
                if not torch.equal(grouped[r], torch.cat([t.view(torch.uint8) for t in rv])):
                    raise RuntimeError(f"{name}: grouped and per-tensor results differ on rank {r}")
            for p in plans:
                p.close()
            for c, ((s, rcv), _, _) in zip(g.comms, made):
                c.free(s)
                c.free(rcv)
    finally:
        g.close()
    return out


def bench_mpi(a, tmp):
    out = {}
    for n in a.mpi_ranks:
        with LocalCluster(n_workers=1, slots_per_worker=n, log_level="warn", log_dir=tmp) as c:
            for name in ("resnet50", "ulysses"):
                if name == "ulysses" and n not in MPI_ULYSSES_RANKS:
                    continue
                sizes, _ = workload(name, n)
                bound_ms = 2 * n * sum(sizes) / HBM_BYTES_PER_S * 1e3
                for mode in ("alltoall", "ialltoall"):
                    reps = []
                    for _ in range(a.reps):
                        st = c.client.invoke(
                            "mpi",
                            "bench-group-alltoall",
                            mpi_world_size=n,
                            input_data=f"{mode};{a.steps};{','.join(map(str, sizes))}",
                            timeout=INVOKE_TIMEOUT_S,
                        )
                        res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
                        if any(m.get("returnValue", 0) != 0 for m in res):
                            raise RuntimeError(f"bench-group-alltoall {mode} on {n} ranks failed: {res}")
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
    ap.add_argument("--mpi-ranks", type=int, nargs="+", default=list(RANKS), help="world sizes of the MPI comparison")
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
