"""Grouped broadcast and grouped all-reduce on sub-communicators, on the 214
ResNet-50 gradient tensors (fp32, 97.6 MiB), ranks sharing cuda:0.

  (a) broadcast from rank 0: 214 `broadcast` calls per rank (bcast_loop)
      against one `broadcast_many` of the list (bcast_many), at 2, 4 and 8
      ranks.  The HBM lower bound of one step is n * S / 3.35 TB/s (H100 SXM
      data-sheet bandwidth, S the list's bytes): every rank but the root
      writes S and the root's S is read; the fraction of it is reported, not
      a target.
  (b) a world of 4 split into two children of 2 ([0, 1] and [2, 3]): per
      tensor `all_reduce` on the children (sub_ar_loop) against one
      `all_reduce_many` per child (sub_ar_many).

Both are measured twice:
  * through MPI: the `bench-group-bcast` function of faabric_worker on one
    worker process whose ranks share cuda:0, as 214 MPI_Bcast against
    MPI_Ibcast x214 + MPI_Waitall, and 214 MPI_Allreduce against
    MPI_Iallreduce x214 + MPI_Waitall on the MPI_Comm_split halves of a world
    of 4 (wall-clock ms per step on rank 0, µs per call = ms per step / 214,
    and rank 0's launches per step on the communicator of the call);
  * on the device layer, the calls those MPI paths issue, on a LocalGroup:
    ms per step (CUDA events), device launches per step per rank (the
    communicators' stats), and host µs per call (wall time to issue one step,
    divided by the calls it replaces).
The card's name and power limit are read in the same run.

    python scripts/bench_group_bcast.py [--steps 20] [--warmup 5] [--reps 3] [--json out.json] [--no-mpi]
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


def card() -> str:
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


def tensors(c):
    """The 214 tensors as 16-byte aligned views of one heap buffer."""
    sizes = resnet50_grad_sizes()
    pad = [(s + 3) // 4 * 4 for s in sizes]
    buf = c.empty(sum(pad), torch.float32)
    buf.copy_(torch.arange(sum(pad), device=buf.device, dtype=torch.float32) % 251)
    views, o = [], 0
    for s, p in zip(sizes, pad):
        views.append(buf[o : o + s])
        o += p
    return buf, views


def loop(g, views, call):
    """Tensor i on every rank before tensor i+1 (stream-ordered barriers
    between ranks sharing a GPU)."""
    cur = torch.cuda.current_stream()
    for st in g.streams:
        st.wait_stream(cur)
    for i in range(len(views[0])):
        for r, c in enumerate(g.comms):
            with torch.cuda.stream(g.streams[r]):
                call(c, views[r][i], g.streams[r])


def measure(groups, fn, steps, warmup, calls):
    """(ms per step, launches per step per rank, host µs per replaced call)"""
    cur = torch.cuda.current_stream()
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    comms = [c for g in groups for c in g.comms]
    l0 = [c.stats()["launches"] for c in comms]
    start = torch.cuda.Event(enable_timing=True)
    end = torch.cuda.Event(enable_timing=True)
    start.record(cur)
    host = 0.0
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        host += time.perf_counter() - t0
    for g in groups:
        for st in g.streams:
            cur.wait_stream(st)
    end.record(cur)
    end.synchronize()
    for g in groups:
        if g.check_errors() != [0] * g.size:
            raise RuntimeError("device watchdog fired")
    launches = max(c.stats()["launches"] - b for c, b in zip(comms, l0)) / steps
    return start.elapsed_time(end) / steps, launches, host / steps / calls * 1e6


def bench_bcast(n, a):
    g = LocalGroup(n, devices=[0] * n, heapBytes=256 << 20, stageBytes=8 << 20, timeoutMs=20000)
    out = {}
    try:
        bufs = [tensors(c) for c in g.comms]
        views = [v for _, v in bufs]
        nbytes = sum(t.numel() * 4 for t in views[0])
        bound_ms = n * nbytes / HBM_BYTES_PER_S * 1e3
        modes = {
            "bcast_loop": lambda: loop(g, views, lambda c, t, st: c.broadcast(t, root=0, stream=st)),
            "bcast_many": lambda: g.run(lambda c, r, st: c.broadcast_many(views[r], root=0)),
        }
        for mode, fn in modes.items():
            reps = [measure([g], fn, a.steps, a.warmup, len(views[0])) for _ in range(a.reps)]
            ms = sorted(x[0] for x in reps)
            out[mode] = dict(
                ms_per_step=[round(x, 4) for x in ms],
                launches_per_step=reps[0][1],
                host_us_per_call=round(sorted(x[2] for x in reps)[len(reps) // 2], 2),
                hbm_bound_fraction=round(bound_ms / ms[len(ms) // 2], 3),
            )
            print(json.dumps(dict(ranks=n, mode=mode, mib=round(nbytes / 2**20, 1), **out[mode])), flush=True)
        for c, (buf, _) in zip(g.comms, bufs):
            c.free(buf)
    finally:
        g.close()
    return out


def bench_sub(a):
    g = LocalGroup(4, devices=[0] * 4, heapBytes=256 << 20, stageBytes=8 << 20, timeoutMs=20000)
    out = {}
    try:
        bufs = [tensors(c) for c in g.comms]
        views = [v for _, v in bufs]
        subs = [g.subset([0, 1]), g.subset([2, 3])]
        sviews = [[views[m] for m in s.members] for s in subs]

        def sub_loop():
            for s, v in zip(subs, sviews):
                loop(s, v, lambda c, t, st: c.all_reduce(t, stream=st))

        def sub_many():
            for s, v in zip(subs, sviews):
                s.run(lambda c, r, st: c.all_reduce_many(v[r]))

        for mode, fn in (("sub_ar_loop", sub_loop), ("sub_ar_many", sub_many)):
            reps = [measure(subs, fn, a.steps, a.warmup, len(views[0])) for _ in range(a.reps)]
            out[mode] = dict(
                ms_per_step=sorted(round(x[0], 4) for x in reps),
                launches_per_step=reps[0][1],
                host_us_per_call=round(sorted(x[2] for x in reps)[len(reps) // 2], 2),
            )
            print(json.dumps(dict(ranks="4 as 2x2", mode=mode, **out[mode])), flush=True)
        for s in subs:
            s.close()
        for c, (buf, _) in zip(g.comms, bufs):
            c.free(buf)
    finally:
        g.close()
    return out


def bench_mpi(a, tmp):
    """Rows of the MPI comparison: (ranks, mode) -> [rank 0's result per rep]"""
    counts = ",".join(str(s) for s in resnet50_grad_sizes())
    out = {}
    cases = [(n, m) for n in (2, 4, 8) for m in ("bcast", "ibcast")] + [(4, "sub-allreduce"), (4, "sub-iallreduce")]
    for n in a.mpi_ranks:
        with LocalCluster(n_workers=1, slots_per_worker=n, log_level="warn", log_dir=tmp) as c:
            for ranks, mode in cases:
                if ranks != n:
                    continue
                reps = []
                for _ in range(a.reps):
                    st = c.client.invoke(
                        "mpi", "bench-group-bcast", mpi_world_size=n, input_data=f"{mode};{a.steps};{counts}", timeout=900
                    )
                    res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
                    if any(m.get("returnValue", 0) != 0 for m in res):
                        raise RuntimeError(f"bench-group-bcast {mode} on {n} ranks failed: {res}")
                    reps.append(json.loads(res[0]["output_data"]))
                ms = sorted(r["ms_per_step"] for r in reps)
                row = dict(
                    ms_per_step=[round(x, 3) for x in ms],
                    us_per_call=round(sorted(r["us_per_call"] for r in reps)[len(reps) // 2], 2),
                    launches_per_step=reps[0]["launches_per_step"],
                )
                if mode.endswith("bcast"):
                    bound_ms = n * sum(resnet50_grad_sizes()) * 4 / HBM_BYTES_PER_S * 1e3
                    row["hbm_bound_fraction"] = round(bound_ms / ms[len(ms) // 2], 3)
                out[f"{ranks}/{mode}"] = row
                print(json.dumps(dict(ranks=ranks, mode=f"mpi {mode}", **row)), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", type=str, default=None)
    ap.add_argument("--no-mpi", action="store_true", help="only the device-layer calls")
    ap.add_argument("--no-device", action="store_true", help="only the MPI calls")
    ap.add_argument("--mpi-ranks", type=int, nargs="+", default=[2, 4, 8], help="world sizes of the MPI comparison")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    the_card = card()
    print(f"# {the_card}", flush=True)
    results = {}
    if not a.no_mpi:
        with tempfile.TemporaryDirectory() as d:
            results["mpi"] = bench_mpi(a, Path(d))
    if not a.no_device:
        results.update({f"bcast/{n}": bench_bcast(n, a) for n in (2, 4, 8)})
        results["subcomm/2x2"] = bench_sub(a)
    if a.json:
        Path(a.json).write_text(json.dumps(dict(card=the_card, results=results), indent=1))


if __name__ == "__main__":
    main()
