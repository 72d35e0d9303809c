"""Device-side timing, clock sampling and structured step logging.

The reference only prints cumulative wall-clock per epoch (train.py:131-137).  For a
multi-GPU trainer numbers must be taken on the device (CUDA events on the launching
stream), reduced as MAX over ranks, and accompanied by the SM clocks seen during the
timed region.
"""
from __future__ import annotations

import json
import subprocess
import sys
import threading
import time
from statistics import median

import torch


class CudaTimer:
    """CUDA-event stopwatch; falls back to perf_counter on CPU."""

    def __init__(self, device=None):
        self.cuda = torch.cuda.is_available() and (device is None or torch.device(device).type == "cuda")
        self._t0 = None
        if self.cuda:
            self._e0 = torch.cuda.Event(enable_timing=True)
            self._e1 = torch.cuda.Event(enable_timing=True)

    def start(self, stream=None):
        if self.cuda:
            torch.cuda.synchronize()
            self._e0.record(stream)
        else:
            self._t0 = time.perf_counter()

    def stop(self, stream=None) -> float:
        """elapsed milliseconds"""
        if self.cuda:
            self._e1.record(stream)
            torch.cuda.synchronize()
            return self._e0.elapsed_time(self._e1)
        return (time.perf_counter() - self._t0) * 1e3


def max_over_ranks(value: float, device=None) -> float:
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return value
    dev = device if device is not None else ("cuda" if dist.get_backend() == "nccl" else "cpu")
    t = torch.tensor([value], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


_QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
          "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
          "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")


class ClockSampler:
    """Samples SM clocks / power / throttle reasons while a timed region runs (the clocks DURING the timed
    region, not before or after it).  Preferred source: NVML in-process (a thread polling every ``period_ms``; works for regions of a few
    milliseconds - the driver times 20 steps of ~0.1 ms); fallback: an ``nvidia-smi -lms`` child process, which needs
    ~100 ms to deliver its first line."""

    _REASONS = (("hw_slowdown", 0x8), ("hw_thermal_slowdown", 0x40), ("sw_thermal_slowdown", 0x20), ("sw_power_cap", 0x4))

    def __init__(self, gpu_index: int = 0, period_ms: int = 100):
        self.gpu_index, self.period_ms = gpu_index, period_ms
        self.proc, self.lines, self._thr = None, [], None
        self._nvml, self._stop, self._samples = None, threading.Event(), []

    # ---- NVML path
    def _nvml_start(self) -> bool:
        try:
            import pynvml

            pynvml.nvmlInit()
            h = pynvml.nvmlDeviceGetHandleByIndex(self.gpu_index)
            mx = float(pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM))
            self._nvml = (pynvml, h, mx)
        except Exception:
            self._nvml = None
            return False

        def pump():
            pynvml, h, mx = self._nvml
            period = max(self.period_ms, 2) / 1e3
            while not self._stop.is_set():
                try:
                    sm = float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM))
                    pw = pynvml.nvmlDeviceGetPowerUsage(h) / 1e3
                    rs = int(pynvml.nvmlDeviceGetCurrentClocksThrottleReasons(h))
                    self._samples.append((sm, mx, pw, rs))
                except Exception:
                    pass
                self._stop.wait(period)

        self._thr = threading.Thread(target=pump, daemon=True)
        self._thr.start()
        return True

    def sample_now(self):
        """one synchronous NVML sample from the calling thread (the bench calls this while a timed block is still in flight on
        the device: the polling thread competes with the step loop for the GIL and may get few turns in a 2 ms region)"""
        if self._nvml is None:
            return
        try:
            pynvml, h, mx = self._nvml
            self._samples.append((float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)), mx,
                                  pynvml.nvmlDeviceGetPowerUsage(h) / 1e3, int(pynvml.nvmlDeviceGetCurrentClocksThrottleReasons(h))))
        except Exception:
            pass

    def __enter__(self):
        if self._nvml_start():
            return self
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={_QUERY}", "--format=csv,noheader,nounits",
                 "-i", str(self.gpu_index), "-lms", str(self.period_ms)],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self._thr = threading.Thread(target=self._pump, daemon=True)
            self._thr.start()
        except Exception:
            self.proc = None
        return self

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def __exit__(self, *exc):
        self._stop.set()
        if self._nvml is not None and self._thr is not None:
            self._thr.join(timeout=2)
        if self.proc is not None:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=5)
            except Exception:
                self.proc.kill()
        return False

    def summary(self) -> dict:
        sm, mx, reasons, power = [], [], set(), []
        if self._nvml is not None:
            for c, m, p, r in self._samples:
                sm.append(c); mx.append(m); power.append(p)
                for name, bit in self._REASONS:
                    if r & bit:
                        reasons.add(name)
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2])); power.append(float(f[3]))
            except ValueError:
                continue
            for name, val in zip(names, f[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        busy = [c for c, p in zip(sm, power) if p > 0.3 * max(power)] or sm
        return {"sm_mhz": median(busy), "sm_max_mhz": max(mx), "reasons": sorted(reasons),
                "samples": len(sm), "power_w_max": max(power), "source": "nvml" if self._nvml is not None else "nvidia-smi"}


class StepLogger:
    """Rank-0 JSON-lines metrics (samples/s, step ms, exposed comm ms, accuracy, loss)."""

    def __init__(self, path=None, rank: int = 0, stream=None):
        self.rank = rank
        self.fh = open(path, "a") if (path and rank == 0) else None
        self.stream = stream if stream is not None else sys.stdout

    def log(self, **fields):
        if self.rank != 0:
            return
        rec = {"ts": time.time(), **fields}
        line = json.dumps(rec)
        if self.fh:
            self.fh.write(line + "\n")
            self.fh.flush()
        else:
            print(line, file=self.stream, flush=True)

    def close(self):
        if self.fh:
            self.fh.close()
