"""Multi-process wiring (Communicator::createIpc): two processes on one GPU,
each creating its communicator through init_from_env, exchange heap handles
over the bootstrap socket and run collectives and point-to-point against closed
forms.  Stream-ordered synchronisation keeps every kernel free of waits on the
other process's kernels, so the processes need not run concurrently on the GPU."""

import os
import subprocess
import sys
import uuid
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]

pytestmark = pytest.mark.gpu

CHILD = r"""
import sys
import torch
from faabric_b200.parallel import init_from_env

c = init_from_env(useVmm=int(sys.argv[1]), useMulticast=0, streamSync=1, timeoutMs=5000,
                  heapBytes=64 << 20, stageBytes=4 << 20)
r, n = c.rank, c.size
print("backing", c.backing, flush=True)
assert n == 2 and c.stream_sync
dev = f"cuda:{c.device}"
st = torch.cuda.Stream()
checks = []
with torch.cuda.stream(st):
    # 4 KB: LL-sized, run as one-shot in stream mode; 80 KB one-shot; 1.2 MB two-shot
    for numel, algo in ((1000, "oneshot"), (20000, "oneshot"), (300000, "twoshot")):
        a = c.empty(numel, torch.int32)
        a.copy_(torch.arange(numel, dtype=torch.int32, device=dev) + r)
        out = c.empty(numel, torch.int32)
        c.all_reduce(a, out, stream=st)
        assert c.last_algo == algo, (numel, c.last_algo)
        checks.append((out, n * torch.arange(numel, dtype=torch.int32) + n * (n - 1) // 2))
    g = c.empty(4096, torch.int32)
    g.copy_(torch.arange(4096, dtype=torch.int32, device=dev) + 1000 * r)
    gout = torch.empty(n * 4096, dtype=torch.int32, device=dev)
    c.all_gather(g, gout, stream=st)
    checks.append((gout, torch.cat([torch.arange(4096, dtype=torch.int32) + 1000 * p for p in range(n)])))
    b = c.empty(5000, torch.int32)
    b.copy_(torch.arange(5000, dtype=torch.int32, device=dev) if r == 0 else torch.full((5000,), -1, dtype=torch.int32, device=dev))
    c.broadcast(b, root=0, stream=st)
    checks.append((b, torch.arange(5000, dtype=torch.int32)))
    msg = torch.arange(70000, dtype=torch.int32, device=dev) + 7 * (r + 1)
    got = torch.zeros(70000, dtype=torch.int32, device=dev)
    if r == 0:
        c.send(msg, 1, stream=st)
        c.recv(got, 1, stream=st)
    else:
        c.recv(got, 0, stream=st)
        c.send(msg, 0, stream=st)
    checks.append((got, torch.arange(70000, dtype=torch.int32) + 7 * (2 - r)))
st.synchronize()
assert c.check_error(st) == 0
for i, (have, want) in enumerate(checks):
    assert torch.equal(have.cpu(), want), i
c.close()
print("ok", flush=True)
"""


@pytest.mark.parametrize("use_vmm, backing", [(1, "vmm-ipc"), (0, "cuda-ipc")])
def test_two_processes_on_one_gpu(use_vmm, backing):
    job = f"ipc-test-{uuid.uuid4().hex[:12]}"
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK="0", FAABRIC_JOB_ID=job)
        env["PYTHONPATH"] = os.pathsep.join([str(ROOT)] + [p for p in [env.get("PYTHONPATH")] if p])
        procs.append(
            subprocess.Popen(
                [sys.executable, "-c", CHILD, str(use_vmm)],
                cwd=ROOT,
                env=env,
                stdout=subprocess.PIPE,
                stderr=subprocess.STDOUT,
                text=True,
            )
        )
    outs = []
    try:
        for p in procs:
            outs.append(p.communicate(timeout=180)[0])
    except subprocess.TimeoutExpired:
        for p in procs:
            p.kill()
        outs = [p.communicate()[0] for p in procs]
        pytest.fail("IPC ranks timed out:\n" + "\n".join(f"rank {r}:\n{o}" for r, o in enumerate(outs)))
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    for rank, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, f"rank {rank}:\n{out}"
        assert f"backing {backing}\n" in out, f"rank {rank}:\n{out}"
        assert out.rstrip().endswith("ok"), f"rank {rank}:\n{out}"
