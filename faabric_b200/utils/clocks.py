"""nvidia-smi clock / throttle sampling during a timed region (profiling
recipe: clocks line)."""

from __future__ import annotations

import shutil
import statistics
import subprocess
import time

_QUERY = (
    "index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
    "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
    "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
)


class ClockSampler:
    def __init__(self, period_ms: int = 100, gpu_index: int | None = None):
        self.period_ms = period_ms
        self.gpu_index = gpu_index
        self.proc = None

    def start(self):
        if shutil.which("nvidia-smi") is None:
            return self
        cmd = ["nvidia-smi", f"--query-gpu={_QUERY}", "--format=csv,noheader,nounits", "-lms", str(self.period_ms)]
        if self.gpu_index is not None:
            cmd += ["-i", str(self.gpu_index)]
        try:
            self.proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except Exception:
            self.proc = None
        return self

    def stop(self) -> dict:
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        time.sleep(self.period_ms / 1000.0)
        self.proc.terminate()
        try:
            out, _ = self.proc.communicate(timeout=5)
        except Exception:
            self.proc.kill()
            out = ""
        sm, mx, power = [], [], []
        reasons = set()
        for line in out.splitlines():
            parts = [p.strip() for p in line.split(",")]
            if len(parts) < 9:
                continue
            try:
                sm.append(float(parts[1]))
                mx.append(float(parts[2]))
                power.append(float(parts[3]))
            except ValueError:
                continue
            names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
            for name, v in zip(names, parts[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        # "under load" = samples in the top half of the observed power range
        return {
            "sm_mhz": statistics.median(sm),
            "sm_max_mhz": max(mx),
            "power_w_max": max(power),
            "reasons": sorted(reasons),
            "samples": len(sm),
        }
