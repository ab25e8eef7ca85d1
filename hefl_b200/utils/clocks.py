"""Sample SM clocks and throttle reasons during a timed region."""
from __future__ import annotations

import statistics
import threading
import time
from typing import Dict, List, Optional


class ClockSampler:
    def __init__(self, device_index: int = 0, period_s: float = 0.05):
        self.idx = device_index
        self.period = period_s
        self.samples: List[int] = []
        self.reasons: set = set()
        self.max_mhz: Optional[int] = None
        self._stop = threading.Event()
        self._thr: Optional[threading.Thread] = None
        self._nvml = None
        try:
            import pynvml

            pynvml.nvmlInit()
            self._nvml = pynvml
            self._h = pynvml.nvmlDeviceGetHandleByIndex(device_index)
            self.max_mhz = int(pynvml.nvmlDeviceGetMaxClockInfo(self._h, pynvml.NVML_CLOCK_SM))
        except Exception:  # noqa: BLE001 - no NVML on this box
            self._nvml = None

    _REASONS = {
        "hw_slowdown": 0x8, "sw_power_cap": 0x4, "hw_thermal_slowdown": 0x40,
        "sw_thermal_slowdown": 0x20, "hw_power_brake_slowdown": 0x80, "sync_boost": 0x10,
    }

    def _loop(self):
        n = self._nvml
        while not self._stop.is_set():
            try:
                self.samples.append(int(n.nvmlDeviceGetClockInfo(self._h, n.NVML_CLOCK_SM)))
                mask = int(n.nvmlDeviceGetCurrentClocksEventReasons(self._h))
                for name, bit in self._REASONS.items():
                    if mask & bit:
                        self.reasons.add(name)
            except Exception:  # noqa: BLE001
                pass
            self._stop.wait(self.period)

    def start(self):
        if self._nvml is None:
            return self
        self._stop.clear()
        self._thr = threading.Thread(target=self._loop, daemon=True)
        self._thr.start()
        return self

    def stop(self) -> Dict:
        if self._thr is not None:
            self._stop.set()
            self._thr.join(timeout=2)
        med = int(statistics.median(self.samples)) if self.samples else None
        return {"sm_mhz": med, "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons),
                "samples": len(self.samples)}
