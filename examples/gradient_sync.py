"""The headline workload on GPUs: all-reduce the 214 gradient tensors of a
ResNet-50 (int32, SUM) with one fused kernel per tensor, replayed from a CUDA
graph.  Needs H100s:

    python examples/gradient_sync.py                       # 1 GPU
    torchrun --nproc-per-node 8 examples/gradient_sync.py  # one process per GPU
"""

import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import torch  # noqa: E402

from faabric_b200.models import GradientSync, resnet50_grad_sizes  # noqa: E402
from faabric_b200.parallel import init_from_env  # noqa: E402


def main() -> int:
    if not torch.cuda.is_available():
        print("this example needs a CUDA device")
        return 2
    comm = init_from_env()  # rank / world size from the torchrun environment
    sync = GradientSync(comm, resnet50_grad_sizes(), dtype=torch.int32, channels=8, algo="tuned")
    for view in sync.send_views:
        view.fill_(comm.rank + 1)
    sync.step()
    torch.cuda.synchronize()
    expected = comm.size * (comm.size + 1) // 2
    ok = all(int(v[0]) == expected and int(v[-1]) == expected for v in sync.recv_views)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(20):
        sync.step()
    end.record()
    torch.cuda.synchronize()
    if comm.rank == 0:
        print(f"{comm.size} GPUs, {sync.launches_per_step} fused all-reduces per step: {start.elapsed_time(end) / 20:.3f} ms/step, correct={ok}")
    sync.close()
    return 0 if ok else 1


if __name__ == "__main__":
    raise SystemExit(main())
