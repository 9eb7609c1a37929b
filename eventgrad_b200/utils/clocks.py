"""Sample GPU clocks / throttle reasons with nvidia-smi during a timed region
(the clocks DURING the timed region are part of a number)."""
from __future__ import annotations

import statistics
import subprocess
import threading
from typing import Dict, List

_Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
      "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
      "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")


class NvmlClockSampler:
    """In-process NVML poller (nvidia_ml_py): ~2 ms period, so even a 40 ms timed region carries >= 5 samples (the
    nvidia-smi -lms poller of round 1 returned 0 samples at N >= 2).  Only samples taken between mark_begin() and
    stop() count; the handle is looked up by the CUDA device's UUID, so CUDA_VISIBLE_DEVICES remapping is harmless."""

    _BITS = {0x8: "hw_slowdown", 0x40: "hw_thermal_slowdown", 0x20: "sw_thermal_slowdown", 0x4: "sw_power_cap"}

    def __init__(self, cuda_index: int = 0, period_ms: float = 2.0):
        self.idx, self.period = cuda_index, period_ms / 1e3
        self.samples = []
        self._stop = threading.Event()
        self._begin = None
        self._t = None
        self.h = None
        self.nv = None

    def start(self) -> "NvmlClockSampler":
        try:
            import pynvml
            import torch
            pynvml.nvmlInit()
            uuid = str(torch.cuda.get_device_properties(self.idx).uuid)
            try:
                self.h = pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid).encode())
            except Exception:
                self.h = pynvml.nvmlDeviceGetHandleByIndex(self.idx)
            self.nv = pynvml
        except Exception:
            self.nv = None
            return self
        nv, h = self.nv, self.h
        reasons_fn = getattr(nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or \
            getattr(nv, "nvmlDeviceGetCurrentClocksThrottleReasons")

        def pump():
            import time
            while not self._stop.is_set():
                try:
                    self.samples.append((time.perf_counter(), nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM),
                                         nv.nvmlDeviceGetPowerUsage(h) / 1e3, int(reasons_fn(h))))
                except Exception:
                    pass
                time.sleep(self.period)
        self._t = threading.Thread(target=pump, daemon=True)
        self._t.start()
        return self

    def mark_begin(self) -> None:
        import time
        self._begin = time.perf_counter()

    def stop(self) -> Dict:
        import time
        end = time.perf_counter()
        self._stop.set()
        if self.nv is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "samples": 0, "reasons": ["nvml unavailable"]}
        self._t.join(timeout=1)
        t0 = self._begin or 0.0
        inside = [s for s in self.samples if t0 <= s[0] <= end]
        try:
            mx = float(self.nv.nvmlDeviceGetMaxClockInfo(self.h, self.nv.NVML_CLOCK_SM))
        except Exception:
            mx = None
        reasons = set()
        for s in inside:
            for bit, nm in self._BITS.items():
                if s[3] & bit:
                    reasons.add(nm)
        sm = [float(s[1]) for s in inside]
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": mx,
                "power_w_max": max((s[2] for s in inside), default=None),
                "samples": len(sm), "period_ms": self.period * 1e3, "source": "nvml", "reasons": sorted(reasons)}


class ClockSampler:
    def __init__(self, gpu_index: int = 0, period_ms: int = 100):
        self.gpu, self.period = gpu_index, period_ms
        self.proc = None
        self.lines: List[str] = []
        self._t = None

    def start(self) -> "ClockSampler":
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={_Q}", "--format=csv,noheader,nounits",
                 "-i", str(self.gpu), "-lms", str(self.period)],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except (FileNotFoundError, OSError):
            self.proc = None
            return self

        def pump():
            for ln in self.proc.stdout:
                self.lines.append(ln.strip())
        self._t = threading.Thread(target=pump, daemon=True)
        self._t.start()
        return self

    def stop(self) -> Dict:
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, pw = [], [], []
        reasons = set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2])); pw.append(float(f[3]))
            except ValueError:
                continue
            for nm, v in zip(names, f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        return {"sm_mhz": statistics.median(sm) if sm else None,
                "sm_max_mhz": max(mx) if mx else None,
                "power_w_max": max(pw) if pw else None,
                "samples": len(sm), "reasons": sorted(reasons)}


class NvlinkCounters:
    """Hardware NVLink byte counters of one GPU through NVML (cumulative over all links, scope id = all links):
    DATA = payload bytes, RAW = payload + protocol overhead.  `read()` returns a dict of byte counts; take the
    difference around a timed region to MEASURE the NVLink traffic of a kernel sequence instead of inferring it."""

    def __init__(self, cuda_index: int = 0):
        self.ok = False
        try:
            import pynvml
            import torch
            pynvml.nvmlInit()
            uuid = str(torch.cuda.get_device_properties(cuda_index).uuid)
            try:
                self.h = pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid).encode())
            except Exception:
                self.h = pynvml.nvmlDeviceGetHandleByIndex(cuda_index)
            self.nv = pynvml
            self.ids = {"data_tx": pynvml.NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX,
                        "data_rx": pynvml.NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_RX,
                        "raw_tx": pynvml.NVML_FI_DEV_NVLINK_THROUGHPUT_RAW_TX,
                        "raw_rx": pynvml.NVML_FI_DEV_NVLINK_THROUGHPUT_RAW_RX}
            self.ok = self.read() is not None
        except Exception:
            self.ok = False

    def read(self):
        try:
            nv = self.nv
            # scopeId UINT_MAX = aggregate over all links of the device
            req = [(fid, 0xFFFFFFFF) for fid in self.ids.values()]
            try:
                vals = nv.nvmlDeviceGetFieldValues(self.h, req)
            except Exception:
                vals = nv.nvmlDeviceGetFieldValues(self.h, list(self.ids.values()))
            out = {}
            for name, v in zip(self.ids, vals):
                if v.nvmlReturn != 0:
                    return None
                out[name] = int(v.value.ullVal) * 1024          # counters are in KiB
            return out
        except Exception:
            return None
