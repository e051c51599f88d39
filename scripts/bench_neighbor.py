"""Grouped neighbourhood all-to-all (the staged-pull device path behind
neighbor_all_to_all_many and its plans), ranks sharing cuda:0 at 2, 4 and 8
ranks, on two workloads:

  (a) halo: a 2-D periodic 4-neighbour exchange (left, right, down, up) on a
      2x1, 2x2 or 4x2 process grid, five fp32 fields per step, one
      all-to-all item per field, at face sizes of 16 KiB and 1 MiB.  The 2x1
      grid has multi-edges (left and right are the same rank) and self-edges
      (down and up are the rank itself).
  (b) ring: a directed ring, one 8 MiB block per rank per step, where
      bandwidth and the staging copy dominate.

Device-layer arms, on a LocalGroup: one `neighbor_all_to_all_many` of the
step's list (many: its segment table is built and uploaded every step), and
one `neighbor_all_to_all_group` launch of a plan prepared once (plan).  MPI
arms, through the `bench-neighbor` function of faabric_worker on one worker
process whose ranks share cuda:0, per step: an MPI_Isend per out-edge and an
MPI_Irecv per in-edge of every field plus MPI_Waitall (mpi p2p: what programs
write without neighbourhood collectives; self-edges are a device copy), one
blocking MPI_Neighbor_alltoall per field (mpi blocking), and one
MPI_Ineighbor_alltoall per field plus MPI_Waitall (mpi burst); wall-clock ms
per step on rank 0, at MPI_RANKS (see there).  Every invocation is bounded
at 180 s.  Reported:
ms per step from CUDA events (min / median / max over repetitions), device
launches per step per rank (the communicators' stats), and the fraction of
the HBM bound: the bytes the staged design moves (every staged block read
from send and written to staging, every pulled block read from staging and
written to recv) over 3.35 TB/s (H100 SXM data-sheet bandwidth), over the
median.  It is a fraction, not a target.  Each arm's outputs are checked
against the exchange the graph defines before its numbers are printed.  The
card's name and power limit are read in the same run.

    python scripts/bench_neighbor.py [--steps 20] [--warmup 3] [--reps 3] [--json out.json] [--no-mpi]
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

import torch  # noqa: E402

from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import neighbor_in_edges  # noqa: E402
from faabric_b200.runtime import LocalCluster  # noqa: E402

INVOKE_TIMEOUT_S = 180
# As the other grouped benchmarks: the MPI arms run at 2 ranks.  At 4 ranks
# sharing one H100 the first MPI_Isend / MPI_Irecv halo invocation did not
# finish within 180 s (docs/next_steps.md).
MPI_RANKS = (2,)
MPI_MODES = ("p2p", "blocking", "burst")

HBM_BYTES_PER_S = 3.35e12
RANKS = (2, 4, 8)
GRIDS = {2: (2, 1), 4: (2, 2), 8: (4, 2)}
FIELDS = 5
FACES = {"halo16k": 16 << 10, "halo1m": 1 << 20}
RING_BYTES = 8 << 20


def card() -> str:
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


def halo_graph(n):
    px, py = GRIDS[n]
    nbrs = []
    for r in range(n):
        x, y = r % px, r // px
        nbrs.append([(x - 1) % px + y * px, (x + 1) % px + y * px, x + (y - 1) % py * px, x + (y + 1) % py * px])
    return nbrs, nbrs


def ring_graph(n):
    return [[(r - 1) % n] for r in range(n)], [[(r + 1) % n] for r in range(n)]


def workloads(n):
    """name: (sources, destinations, bytes per block, items per step)"""
    out = {name: (*halo_graph(n), face, FIELDS) for name, face in FACES.items()}
    out["ring8m"] = (*ring_graph(n), RING_BYTES, 1)
    return out


def buffers(g, dst, edges, block, items):
    """Every rank's send and recv tensors of each item (fp32), the sends
    filled with values unique to (rank, item, element)"""
    elems = block // 4
    sends, recvs, bases = [], [], []
    for r, c in enumerate(g.comms):
        s = c.empty(items * len(dst[r]) * elems, torch.float32)
        v = c.empty(items * len(edges[r]) * elems, torch.float32)
        s.copy_(torch.arange(s.numel(), device=s.device, dtype=torch.float32) + r * 1e7)
        v.fill_(-1.0)
        sends.append(list(s.view(items, -1).unbind(0)))
        recvs.append(list(v.view(items, -1).unbind(0)))
        bases.append((s, v))
    torch.cuda.synchronize()
    return sends, recvs, bases


def check(sends, recvs, edges, block):
    """recv block j of rank d is block idx of in-edge j's source's send"""
    e = block // 4
    for d, mine in enumerate(edges):
        for i in range(len(recvs[d])):
            for j, (s, idx) in enumerate(mine):
                if not torch.equal(recvs[d][i][j * e : (j + 1) * e], sends[s][i][idx * e : (idx + 1) * e]):
                    raise RuntimeError(f"rank {d} item {i} block {j} differs from rank {s}'s block {idx}")


def measure(g, fn, steps, warmup):
    """(ms per step, launches per step per rank)"""
    cur = torch.cuda.current_stream()
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    l0 = [c.stats()["launches"] for c in g.comms]
    start = torch.cuda.Event(enable_timing=True)
    end = torch.cuda.Event(enable_timing=True)
    start.record(cur)
    for _ in range(steps):
        fn()
    for st in g.streams:
        cur.wait_stream(st)
    end.record(cur)
    end.synchronize()
    if g.check_errors() != [0] * g.size:
        raise RuntimeError("device watchdog fired")
    launches = max(c.stats()["launches"] - b for c, b in zip(g.comms, l0)) / steps
    return start.elapsed_time(end) / steps, launches


def bench(n, a):
    g = LocalGroup(n, devices=[0] * n, heapBytes=256 << 20, timeoutMs=20000)
    out = {}
    try:
        for name, (src, dst, block, items) in workloads(n).items():
            edges = neighbor_in_edges(src, dst)
            # a topology is set once per communicator: one subset per graph
            sub = g.subset(list(range(n)))
            try:
                sub.set_neighbors(src, dst)
                sends, recvs, bases = buffers(g, dst, edges, block, items)
                moved = items * block * 2 * (sum(len(d) for d in dst) + sum(len(e) for e in edges))
                bound_ms = moved / HBM_BYTES_PER_S * 1e3
                plans = [c.prepare_neighbor_all_to_all_group(sends[r], recvs[r]) for r, c in enumerate(sub.comms)]
                modes = {
                    "many": lambda: sub.run(lambda c, r, st: c.neighbor_all_to_all_many(sends[r], recvs[r])),
                    "plan": lambda: sub.run(lambda c, r, st: c.neighbor_all_to_all_group(plans[r])),
                }
                for mode, fn in modes.items():
                    for rv in recvs:
                        for t in rv:
                            t.fill_(-1.0)
                    reps = [measure(sub, fn, a.steps, a.warmup) for _ in range(a.reps)]
                    check(sends, recvs, edges, block)
                    ms = sorted(x[0] for x in reps)
                    r = dict(
                        ms_per_step=dict(min=round(ms[0], 4), median=round(ms[len(ms) // 2], 4), max=round(ms[-1], 4)),
                        launches_per_step=reps[0][1],
                        hbm_bound_fraction=round(bound_ms / ms[len(ms) // 2], 3),
                    )
                    out[f"{name}/{mode}"] = r
                    line = dict(ranks=n, workload=name, mode=mode, block_kib=block >> 10, items=items, **r)
                    print(json.dumps(line), flush=True)
                for p in plans:
                    p.close()
                for c, (s, v) in zip(g.comms, bases):
                    c.free(s)
                    c.free(v)
            finally:
                sub.close()
    finally:
        g.close()
    return out


def bench_mpi(n, a, tmp):
    out = {}
    with LocalCluster(n_workers=1, slots_per_worker=n, log_level="warn", log_dir=tmp) as c:
        for name, (src, dst, block, items) in workloads(n).items():
            moved = items * block * 2 * (sum(len(d) for d in dst) + sum(len(s) for s in src))
            bound_ms = moved / HBM_BYTES_PER_S * 1e3
            graph = "ring" if name.startswith("ring") else "halo"
            for mode in MPI_MODES:
                reps = []
                for _ in range(a.reps):
                    st = c.client.invoke(
                        "mpi",
                        "bench-neighbor",
                        mpi_world_size=n,
                        input_data=f"{mode};{a.steps};{graph};{block};{items}",
                        timeout=INVOKE_TIMEOUT_S,
                    )
                    res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
                    if any(m.get("returnValue", 0) != 0 for m in res):
                        raise RuntimeError(f"bench-neighbor {mode} {name} on {n} ranks failed: {res}")
                    reps.append(json.loads(res[0]["output_data"]))
                ms = sorted(x["ms_per_step"] for x in reps)
                r = dict(
                    ms_per_step=dict(min=round(ms[0], 4), median=round(ms[len(ms) // 2], 4), max=round(ms[-1], 4)),
                    launches_per_step=reps[0]["launches_per_step"],
                    hbm_bound_fraction=round(bound_ms / ms[len(ms) // 2], 3),
                )
                out[f"{name}/mpi {mode}"] = r
                line = dict(ranks=n, workload=name, mode=f"mpi {mode}", block_kib=block >> 10, items=items, **r)
                print(json.dumps(line), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ranks", type=int, nargs="*", default=list(RANKS))
    ap.add_argument("--json", type=str, default=None)
    ap.add_argument("--no-mpi", action="store_true")
    a = ap.parse_args()
    the_card = card()
    print(json.dumps(dict(card=the_card)), flush=True)
    results = {}
    with tempfile.TemporaryDirectory() as tmp:
        for n in a.ranks:
            results[n] = bench(n, a)
            if not a.no_mpi and n in MPI_RANKS:
                results[n].update(bench_mpi(n, a, tmp))
    if a.json:
        Path(a.json).write_text(json.dumps(dict(card=the_card, results=results), indent=1))


if __name__ == "__main__":
    main()
