"""nvidia-smi clock / throttle sampler used while a timed region runs (read-only queries)."""
from __future__ import annotations

import shutil
import statistics
import subprocess
import threading
from typing import Dict, List, Optional

_QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
          "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")


class ClockSampler:
    def __init__(self, gpu_index: int = 0, period_ms: int = 25):
        self.gpu_index, self.period_ms = gpu_index, period_ms
        self.lines: List[str] = []
        self.proc: Optional[subprocess.Popen] = None
        self.thread: Optional[threading.Thread] = None

    def start(self) -> "ClockSampler":
        exe = shutil.which("nvidia-smi")
        if not exe:
            return self
        self.proc = subprocess.Popen([exe, f"--query-gpu={_QUERY}", "--format=csv,noheader,nounits", "-i", str(self.gpu_index),
                                      "-lms", str(self.period_ms)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        self.thread = threading.Thread(target=self._pump, daemon=True)
        self.thread.start()
        return self

    def _pump(self):
        assert self.proc and self.proc.stdout
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self) -> Dict[str, object]:
        if self.proc:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=3)
            except Exception:
                self.proc.kill()
        sm, mx, pw = [], [], []
        reasons = set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            parts = [p.strip() for p in ln.split(",")]
            if len(parts) < 9:
                continue
            try:
                sm.append(float(parts[1]))
                mx.append(float(parts[2]))
                pw.append(float(parts[3]))
            except ValueError:
                continue
            for nm, val in zip(names, parts[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(nm)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(mx), "power_w_max": max(pw), "reasons": sorted(reasons),
                "samples": len(sm)}
