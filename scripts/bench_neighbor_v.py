"""MPI neighbourhood v-collectives (the staged-pull v kernel behind
MPI_Neighbor_alltoallv and MPI_Ineighbor_alltoallv bursts) through the
`bench-neighbor-v` function of faabric_worker, on one worker process whose
ranks share cuda:0.  Two workloads on the periodic 4-neighbour halo of a
2x1, 2x2 or 4x2 process grid (left, right, down, up), five fp32 fields per
step:

  (a) irregular: the face rank r sends on out-edge k has face * (1 + (r + k)
      % 4) / 4 bytes, so every edge of a rank has its own size, and the two
      ends of a rank pair differ.  Arms, per step: an MPI_Isend per out-edge
      and an MPI_Irecv per in-edge of every field plus MPI_Waitall (p2p: what
      programs write without the v calls), one blocking
      MPI_Neighbor_alltoallv per field (blocking: one host agreement and one
      launch each), one MPI_Ineighbor_alltoallv per field plus MPI_Waitall
      (burst: one agreement and one launch per step).
  (b) equal: every face the same size; the v burst against an
      MPI_Ineighbor_alltoall burst on the same data (equal), which shows what
      the v burst's host agreement costs.

Every invocation is bounded at 180 s, the p2p arm above 2 ranks at
P2P_TIMEOUT_S: at 4 ranks sharing one H100 the first MPI_Isend / MPI_Irecv
halo invocation of the equal-block benchmark did not finish within 180 s
(docs/next_steps.md), and an arm that does not finish is reported as such.
Each arm runs on a worker of its own: a worker keeps every MPI world it ran,
device heaps included.  Reported: wall-clock ms per step on rank 0 (min / median / max over
repetitions) and device launches per step on rank 0 (the world device
communicator's and the graph child's stats).  Every rank checks every word it
received against the exchange the graph defines before the numbers count.
The card's name and power limit are read in the same run.

    python scripts/bench_neighbor_v.py [--steps 20] [--reps 3] [--ranks 2 4 8] [--json out.json] [--log-dir d]
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

INVOKE_TIMEOUT_S = 180
P2P_TIMEOUT_S = 40
RANKS = (2, 4, 8)
FIELDS = 5
FACES = (16 << 10, 1 << 20)
ARMS = {"irregular": ("p2p", "blocking", "burst"), "equal": ("burst", "equal")}


def card() -> str:
    r = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
        capture_output=True,
        text=True,
        timeout=30,
    )
    return r.stdout.strip() or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ranks", type=int, nargs="*", default=list(RANKS))
    ap.add_argument("--json", type=str, default=None)
    ap.add_argument("--log-dir", type=str, default=None, help="keep the planner and worker logs here")
    a = ap.parse_args()
    the_card = card()
    print(json.dumps(dict(card=the_card)), flush=True)
    results = []
    with tempfile.TemporaryDirectory() as tmp:
        for n in a.ranks:
            for faces, arms in ARMS.items():
                for face in FACES:
                    for mode in arms:
                        logs = Path(a.log_dir) / f"ranks{n}-{faces}-{face >> 10}k-{mode}" if a.log_dir else Path(tmp)
                        with LocalCluster(n_workers=1, slots_per_worker=n, log_level="warn", log_dir=logs) as c:
                            reps = []
                            limit = P2P_TIMEOUT_S if mode == "p2p" and n > 2 else INVOKE_TIMEOUT_S
                            for _ in range(a.reps):
                                try:
                                    st = c.client.invoke(
                                        "mpi",
                                        "bench-neighbor-v",
                                        mpi_world_size=n,
                                        input_data=f"{mode};{a.steps};{faces};{face};{FIELDS}",
                                        timeout=limit,
                                    )
                                except Exception as e:  # a timeout: reported, not measured
                                    if mode != "p2p":
                                        raise
                                    reps = None
                                    print(json.dumps(dict(ranks=n, faces=faces, face_kib=face >> 10, mode=mode,
                                                          not_finished_in_s=limit, error=str(e)[:200])), flush=True)
                                    break
                                res = sorted(st["messageResults"], key=lambda m: m.get("mpiRank", 0))
                                if any(m.get("returnValue", 0) != 0 for m in res):
                                    raise RuntimeError(f"bench-neighbor-v {mode} {faces} on {n} ranks failed: {res}")
                                reps.append(json.loads(res[0]["output_data"]))
                            if reps is None:
                                results.append(dict(ranks=n, faces=faces, face_kib=face >> 10, mode=mode,
                                                    not_finished_in_s=limit))
                                continue
                            ms = sorted(x["ms_per_step"] for x in reps)
                            line = dict(
                                ranks=n,
                                faces=faces,
                                face_kib=face >> 10,
                                mode=mode,
                                ms_per_step=dict(
                                    min=round(ms[0], 4), median=round(ms[len(ms) // 2], 4), max=round(ms[-1], 4)
                                ),
                                launches_per_step=reps[0]["launches_per_step"],
                            )
                            results.append(line)
                            print(json.dumps(line), flush=True)
    if a.json:
        Path(a.json).write_text(json.dumps(dict(card=the_card, results=results), indent=1))


if __name__ == "__main__":
    main()
