"""Sample SM clocks / throttle reasons while a timed region runs.

Follows the profiling recipe: samples are taken DURING the timed regions and the summary
(median SM MHz under load, max SM MHz, active throttle reasons) is attached to every reported
number.  Timed regions here are tens of milliseconds, far shorter than an ``nvidia-smi -lms``
period, so the primary sampler is an NVML polling thread (``pynvml``, ~1 kHz); ``nvidia-smi``
is the fallback.

``start()`` does all the slow work (``nvmlInit``, handle lookup, thread start) and must be called
well before any timed region — never between a cross-rank barrier and the start event: NVML
calls take tens of milliseconds when eight processes keep the GPUs busy, and the other ranks'
kernels would wait for this rank inside their timed region.  ``pause()`` / ``resume()`` only flip a flag the polling thread reads.
"""
from __future__ import annotations

import shutil
import statistics
import subprocess
import tempfile
import threading
import time
from typing import Dict, List, Optional

_FIELDS = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
           "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
           "clocks_event_reasons.sw_power_cap")
_REASONS = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]

# nvmlClocksEventReasons bit masks (nvml.h)
_NVML_REASON_BITS = {
    "sw_power_cap": 0x4,
    "hw_slowdown": 0x8,
    "sw_thermal_slowdown": 0x20,
    "hw_thermal_slowdown": 0x40,
}

_EMPTY = {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}


def _summary(sm: List[float], sm_max: float, power: List[float], reasons: set, how: str) -> Dict:
    if not sm:
        return dict(_EMPTY, sampler=how)
    lo, hi = (min(power), max(power)) if power else (0.0, 0.0)
    loaded = [c for c, p in zip(sm, power) if p >= lo + 0.5 * (hi - lo)] if power else sm
    loaded = loaded or sm
    return {"sm_mhz": statistics.median(loaded), "sm_max_mhz": sm_max, "power_w_max": hi,
            "reasons": sorted(reasons), "samples": len(sm), "sampler": how}


class ClockSampler:
    """``with``-less start()/stop() sampler for one GPU (by NVML index)."""

    def __init__(self, gpu_index: int = 0, period_ms: float = 1.0, uuid: Optional[str] = None):
        self.gpu_index = gpu_index
        self.uuid = uuid  # "GPU-..." : robust when CUDA and NVML enumerate in different orders
        self.period_s = max(period_ms, 0.2) * 1e-3
        self._thread: Optional[threading.Thread] = None
        self._stop = threading.Event()
        self._active = True
        self._sm: List[float] = []
        self._power: List[float] = []
        self._reasons: set = set()
        self._sm_max = 0.0
        self._proc: Optional[subprocess.Popen] = None
        self._file = None
        self._how = "none"

    # ---- NVML thread ---------------------------------------------------------------
    def _nvml_loop(self, nv, handle) -> None:
        while not self._stop.is_set():
            if not self._active:
                time.sleep(self.period_s)
                continue
            try:
                self._sm.append(float(nv.nvmlDeviceGetClockInfo(handle, nv.NVML_CLOCK_SM)))
                self._power.append(nv.nvmlDeviceGetPowerUsage(handle) / 1000.0)
                try:
                    mask = nv.nvmlDeviceGetCurrentClocksEventReasons(handle)
                except AttributeError:
                    mask = nv.nvmlDeviceGetCurrentClocksThrottleReasons(handle)
                for name, bit in _NVML_REASON_BITS.items():
                    if mask & bit:
                        self._reasons.add(name)
            except Exception:
                pass
            time.sleep(self.period_s)

    def pause(self) -> None:
        self._active = False

    def resume(self) -> None:
        self._active = True

    def start(self, paused: bool = False) -> "ClockSampler":
        self._active = not paused
        try:
            import pynvml as nv

            nv.nvmlInit()
            handle = None
            if self.uuid:
                try:
                    handle = nv.nvmlDeviceGetHandleByUUID(self.uuid.encode() if isinstance(self.uuid, str) else self.uuid)
                except Exception:
                    handle = None
            if handle is None:
                handle = nv.nvmlDeviceGetHandleByIndex(self.gpu_index)
            self._sm_max = float(nv.nvmlDeviceGetMaxClockInfo(handle, nv.NVML_CLOCK_SM))
            self._how = "nvml-thread"
            self._thread = threading.Thread(target=self._nvml_loop, args=(nv, handle), daemon=True)
            self._thread.start()
            return self
        except Exception:
            self._thread = None
        exe = shutil.which("nvidia-smi")
        if exe is None:
            return self
        self._file = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        cmd = [exe, f"--query-gpu={_FIELDS}", "--format=csv,noheader,nounits", "-lms", "20",
               "-i", str(self.gpu_index)]
        try:
            self._proc = subprocess.Popen(cmd, stdout=self._file, stderr=subprocess.DEVNULL)
            self._how = "nvidia-smi"
        except OSError:
            self._proc = None
        return self

    def stop(self) -> Dict:
        if self._thread is not None:
            self._stop.set()
            self._thread.join(timeout=2)
            return _summary(self._sm, self._sm_max, self._power, self._reasons, self._how)
        if self._proc is None:
            return dict(_EMPTY, sampler="none")
        self._proc.terminate()
        try:
            self._proc.wait(timeout=5)
        except subprocess.TimeoutExpired:
            self._proc.kill()
        self._file.flush()
        self._file.seek(0)
        return summarize(self._file.read().splitlines())


def summarize(lines: List[str]) -> Dict:
    """Summarise ``nvidia-smi --query-gpu=<_FIELDS> --format=csv,noheader,nounits`` lines."""
    sm: List[float] = []
    sm_max: List[float] = []
    power: List[float] = []
    reasons = set()
    for line in lines:
        parts = [p.strip() for p in line.split(",")]
        if len(parts) < 8:
            continue
        try:
            sm.append(float(parts[1]))
            sm_max.append(float(parts[2]))
            power.append(float(parts[3]))
        except ValueError:
            continue
        for name, val in zip(_REASONS, parts[4:8]):
            if val.lower().startswith("active"):
                reasons.add(name)
    return _summary(sm, max(sm_max) if sm_max else 0.0, power, reasons, "nvidia-smi")
