"""All-reduce algorithm autotuner and tuning-file tools.

The native communicator picks LL / one-shot / two-shot / NVLS per message size
from a selection table.  This module builds that table from a measured sweep
(``bench.py --mode sweep`` prints one row per size with ``<algo>_us`` columns)
and reads / writes the plain-text tuning file the C++ side loads when
``FAABRIC_TUNING_FILE`` names it (format: ``CommTuning`` in
``csrc/include/faabric/device/communicator.h``)::

    # comment
    set oneShotMaxBytes 262144
    allreduce 32768 ll
    allreduce 1048576 twoshot
    allreduce 18446744073709551615 nvls

The reference has no counterpart (its all-reduce is always reduce + broadcast,
``src/mpi/MpiWorld.cpp:1251-1264``); SURVEY.md §5.6 asks for a thresholds file.

CLI::

    python -m faabric_b200.parallel.autotune --from-json tuning_N8.json --out tuning_N8.txt
    python -m faabric_b200.parallel.autotune --measure --ranks 8 --out tuning_N8.txt   # needs GPUs
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
from pathlib import Path
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

TABLE_ALGOS = ("ll", "oneshot", "twoshot", "nvls")
SETTING_KEYS = (
    "llMaxBytes",
    "oneShotMaxBytes",
    "nvlsMinBytes",
    "nvlsScalarMinBytes",
    "bcast2StepMinBytes",
    "tmaMinBytes",
    "maxBlocks",
    "threads",
    "channels",
)
U64_MAX = (1 << 64) - 1

Table = List[Tuple[int, str]]


def row_times(r: dict) -> Dict[str, float]:
    """Per-algorithm time of one sweep row.  The `auto` column is a second
    sample of whichever algorithm the policy picked: latency samples are
    one-sided noisy, so the smaller of the two stands for that algorithm."""
    cands = {a: float(r[a + "_us"]) for a in TABLE_ALGOS if isinstance(r.get(a + "_us"), (int, float))}
    pick = r.get("auto_pick")
    if pick in cands and isinstance(r.get("auto_us"), (int, float)):
        cands[pick] = min(cands[pick], float(r["auto_us"]))
    return cands


def pick_for(table: Sequence[Tuple[int, str]], nbytes: int) -> Optional[str]:
    """What a table answers for a message of `nbytes` (first range that covers it)."""
    for max_bytes, algo in sorted(table):
        if nbytes <= max_bytes:
            return algo
    return None


def table_from_rows(rows: Iterable[dict], hysteresis: float = 0.03) -> Table:
    """Fastest algorithm per measured size, merged into ``(max_bytes, algo)``
    ranges.  A challenger must beat the algorithm of the previous (smaller)
    size by ``hysteresis`` to take over, which keeps noise from fragmenting the
    table.  The last range is open-ended."""
    table: Table = []
    prev: Optional[str] = None
    for r in sorted(rows, key=lambda r: r["bytes"]):
        cands = row_times(r)
        if not cands:
            continue
        best = min(cands, key=cands.get)
        if prev in cands and cands[prev] <= cands[best] * (1.0 + hysteresis):
            best = prev
        if table and table[-1][1] == best:
            table[-1] = (int(r["bytes"]), best)
        else:
            table.append((int(r["bytes"]), best))
        prev = best
    if table:
        table[-1] = (U64_MAX, table[-1][1])
    return table


def json_table_from_rows(rows: Iterable[dict]) -> List[dict]:
    """The same table as ``table_from_rows`` in the JSON shape of ``tuning_N*.json``."""
    rows = list(rows)
    out = []
    lo = 0
    for max_bytes, algo in table_from_rows(rows):
        inside = [row_times(r)[algo] for r in rows if lo < int(r["bytes"]) <= max_bytes and algo in row_times(r)]
        out.append({"max_bytes": max(int(r["bytes"]) for r in rows) if max_bytes == U64_MAX else max_bytes, "algo": algo,
                    "us": round(min(inside), 2) if inside else None})
        lo = max_bytes
    return out


def format_tuning(table: Sequence[Tuple[int, str]] = (), settings: Optional[Dict[str, int]] = None, comment: str = "") -> str:
    lines = ["# faabric_b200 communicator tuning"]
    if comment:
        lines += ["# " + c for c in comment.splitlines()]
    for k, v in (settings or {}).items():
        if k not in SETTING_KEYS:
            raise ValueError(f"unknown tuning key {k!r}")
        lines.append(f"set {k} {int(v)}")
    for max_bytes, algo in sorted(table):
        if algo not in TABLE_ALGOS:
            raise ValueError(f"unknown all-reduce algorithm {algo!r}")
        lines.append(f"allreduce {int(max_bytes)} {algo}")
    return "\n".join(lines) + "\n"


def parse_tuning(text: str) -> Tuple[Table, Dict[str, int]]:
    """Python mirror of ``CommTuning::parse`` (same grammar, same errors)."""
    table: Table = []
    settings: Dict[str, int] = {}
    for no, raw in enumerate(text.splitlines(), 1):
        tok = raw.split("#", 1)[0].split()
        if not tok:
            continue
        if tok[0] == "allreduce" and len(tok) >= 3 and tok[2] in TABLE_ALGOS:
            table.append((int(tok[1]), tok[2]))
        elif tok[0] == "set" and len(tok) >= 3 and tok[1] in SETTING_KEYS:
            settings[tok[1]] = int(tok[2])
        else:
            raise ValueError(f"tuning file line {no}: cannot parse {raw.strip()!r}")
    return sorted(table), settings


def native_normalise(text: str) -> str:
    """Round-trips ``text`` through the C++ parser (no device needed)."""
    from .. import _lib

    lib = _lib.load()
    buf = C.create_string_buffer(1 << 16)
    rc = lib.fb_tuning_normalise(text.encode(), buf, len(buf))
    if rc < 0:
        raise ValueError(buf.value.decode())
    return buf.value.decode()


def load_json_table(path) -> Table:
    """``tuning_N*.json`` as written by ``bench.py --mode sweep``."""
    t = json.loads(Path(path).read_text())
    table = [(int(e["max_bytes"]), e["algo"]) for e in t["allreduce"]]
    if table:
        table[-1] = (U64_MAX, table[-1][1])
    return table


def write_tuning_file(path, table: Sequence[Tuple[int, str]], settings: Optional[Dict[str, int]] = None, comment: str = "") -> Path:
    p = Path(path)
    p.parent.mkdir(parents=True, exist_ok=True)
    p.write_text(format_tuning(table, settings, comment))
    return p


def measure_allreduce_rows(nranks: int, max_bytes: int = 64 << 20, dtype="float32", iters: int = 50, warmup: int = 5) -> List[dict]:
    """Times every algorithm at sizes 1 KiB..max_bytes (x4 steps) on ``nranks``
    GPUs of this process with CUDA events; each row holds the MAX over ranks."""
    import torch

    from .comm import LocalGroup

    td = getattr(torch, dtype)
    esize = torch.empty(0, dtype=td).element_size()
    group = LocalGroup(nranks, heapBytes=2 * max_bytes + (64 << 20), channels=1)
    try:
        bufs = group.run(lambda c, r, s: (c.empty(max_bytes // esize, td).fill_(1), c.empty(max_bytes // esize, td)))
        group.synchronize()
        algos = ["ll", "oneshot", "twoshot"] + (["nvls"] if group.comms[0].has_multicast else [])
        rows = []
        nbytes = 1024
        while nbytes <= max_bytes:
            numel = nbytes // esize
            row = {"bytes": nbytes}
            for algo in algos:
                if (algo == "ll" and nbytes > 65536) or (algo == "oneshot" and nbytes > (16 << 20)):
                    continue
                n_it = iters if nbytes <= (16 << 20) else max(5, iters // 5)

                def issue(c, r, s, algo=algo, numel=numel):
                    c.all_reduce(bufs[r][0][:numel], bufs[r][1][:numel], algo=algo, stream=s)

                for _ in range(warmup):
                    group.run(issue)
                group.synchronize()
                evs = []
                for r, c in enumerate(group.comms):
                    with torch.cuda.device(c.device):
                        evs.append((torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
                        evs[r][0].record(group.streams[r])
                for _ in range(n_it):
                    group.run(issue)
                for r, c in enumerate(group.comms):
                    with torch.cuda.device(c.device):
                        evs[r][1].record(group.streams[r])
                group.synchronize()
                row[algo + "_us"] = round(max(a.elapsed_time(b) for a, b in evs) * 1000.0 / n_it, 3)
            rows.append(row)
            nbytes *= 4
        if any(group.check_errors()):
            raise RuntimeError(f"device watchdog fired during tuning: {group.check_errors()}")
        return rows
    finally:
        group.close()


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--from-json", help="tuning_N*.json written by bench.py --mode sweep")
    ap.add_argument("--measure", action="store_true", help="measure on the GPUs of this box")
    ap.add_argument("--ranks", type=int, default=0, help="--measure: number of GPUs (default all)")
    ap.add_argument("--max-bytes", type=int, default=64 << 20)
    ap.add_argument("--set", action="append", default=[], metavar="KEY=VALUE", help="extra threshold, e.g. tmaMinBytes=262144")
    ap.add_argument("--out", required=True)
    a = ap.parse_args(argv)
    settings = {}
    for kv in a.set:
        k, v = kv.split("=", 1)
        settings[k] = int(v)
    if a.measure:
        import torch

        n = a.ranks or torch.cuda.device_count()
        table = table_from_rows(measure_allreduce_rows(n, a.max_bytes))
        comment = f"measured on {n} GPUs"
    elif a.from_json:
        table = load_json_table(a.from_json)
        comment = f"from {a.from_json}"
    else:
        ap.error("one of --from-json / --measure is required")
    text = format_tuning(table, settings, comment)
    native_normalise(text)  # the C++ parser must accept what we write
    Path(a.out).write_text(text)
    print(text, end="")
    return 0


if __name__ == "__main__":
    sys.exit(main())
