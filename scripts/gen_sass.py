#!/usr/bin/env python
"""Regenerate profiles/sass/*.sass and MNEMONICS.md: one cuobjdump -sass
listing per kernel family (a representative instantiation each), plus a count
of the memory / synchronisation mnemonics that show what the kernel does on
the wire (peer / multicast loads and stores, reductions, bulk copies, flags)."""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
LIB = ROOT / "faabric_b200" / "lib" / "libfaabric_b200.so"
OUT = ROOT / "profiles" / "sass"

# family -> regex on the MANGLED name (first match is dumped)
FAMILIES = {
    "groupAllReduceKernel_u32_sum_n8": r"groupAllReduceKernelINS_9VecReduceIjLi2ELb0EEELi8E",
    "groupAllReduceKernel_u32_sum_n1": r"groupAllReduceKernelINS_9VecReduceIjLi2ELb0EEELi1E",
    "reduceKernel_u32_sum_n8": r"reduceKernelINS_9VecReduceIjLi2ELb0EEELi8E",
    "llAllReduceKernel_u32_sum_n8": r"llAllReduceKernelINS_9VecReduceIjLi2ELb0EEELi8E",
    "nvlsKernel_f32_add": r"nvlsKernelILi0E",
    "moveKernel_w16_n8": r"moveKernelILi16ELi8E",
    "moveBulkKernel": r"moveBulkKernel",
    "barrierKernel": r"barrierKernel",
    "p2pSendKernel_w16": r"p2pSendKernelILi16E",
    "p2pPullKernel_w16": r"p2pPullKernelILi16E",
    "putSignalKernel_w16": r"putSignalKernelILi16E",
    "waitSignalKernel": r"waitSignalKernel",
    "signalPeersKernel": r"signalPeersKernel",
    "snapshotDiffPushKernel": r"snapshotDiffPushKernel",
    "snapshotApplyKernel": r"snapshotApplyKernel",
    "dirtyScanKernel": r"dirtyScanKernel",
    "chunkRunsKernel": r"chunkRunsKernel",
    "flagsOrKernel": r"flagsOrKernel",
    "statePushDirtyKernel": r"statePushDirtyKernel",
    "pageSyncKernel": r"pageSyncKernel",
    "pagePullKernel": r"pagePullKernel",
    "pageGatherKernel": r"pageGatherKernel",
}
INTERESTING = re.compile(
    r"\b(LDG|STG|REDG|ATOMG|LDGMC|UBLKCP|UTMALDG|UTMASTG|SYNCS|MEMBAR|CCTL|ERRBAR|BAR|LDS|STS|LDGSTS|UTC\w*|LDTM|STTM|S2UR|CS2R|MATCH|VOTE)\b[\.\w]*"
)


def main():
    names = subprocess.run(["cuobjdump", "-elf", str(LIB)], capture_output=True, text=True).stdout
    mangled = sorted(set(re.findall(r"\.text\.(_Z\w+)", names)))
    OUT.mkdir(parents=True, exist_ok=True)
    for old in OUT.glob("*.sass"):
        old.unlink()
    md = ["# Memory / sync SASS mnemonics per kernel family (cuobjdump -sass, sm_90a)", "",
          "Regenerate with `python scripts/gen_sass.py` after a build.  One representative",
          "instantiation per family; counts are static instruction counts.", ""]
    for fam, rx in FAMILIES.items():
        hit = next((m for m in mangled if re.search(rx, m)), None)
        if hit is None:
            print("no kernel for", fam, file=sys.stderr)
            continue
        sass = subprocess.run(["cuobjdump", "-sass", "-fun", hit, str(LIB)], capture_output=True, text=True).stdout
        (OUT / f"{fam}.sass").write_text(sass)
        counts = collections.Counter()
        n_instr = 0
        for line in sass.splitlines():
            m = re.search(r"/\*[0-9a-f]{4}\*/\s+(.*?);", line)
            if not m:
                continue
            n_instr += 1
            body = re.sub(r"^@!?U?P\d+\s+", "", m.group(1).strip())
            op = body.split()[0]
            if INTERESTING.match(op):
                counts[op] += 1
        md.append(f"## {fam}.sass  ({n_instr} instructions, `{hit[:70]}`)")
        for op, c in sorted(counts.items()):
            md.append(f"  {op:<40} {c}")
        md.append("")
    (OUT / "MNEMONICS.md").write_text("\n".join(md))
    print("wrote", len(list(OUT.glob('*.sass'))), "listings")


if __name__ == "__main__":
    main()
