"""Timing hygiene helpers: CUDA events on the launching stream,
synchronise on both sides, max over ranks, L2 flush between iterations, clock sampling."""

from __future__ import annotations

import statistics
import subprocess
import threading
import time
from typing import Callable, Optional

import torch


def max_over_ranks(value: float, comm=None) -> float:
    """Max of a host float over all ranks (control plane; not inside timed regions)."""
    import torch.distributed as dist

    from .._src.comm import get_world

    comm = comm or get_world()
    if comm.Get_size() == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=comm._group)
    return float(t.item())


_l2_buf: Optional[torch.Tensor] = None


def flush_l2(device=None, nbytes: int = 256 << 20) -> None:
    """Write a buffer several times larger than the L2 (50 MB on H100)."""
    global _l2_buf
    if _l2_buf is None or _l2_buf.numel() < nbytes:
        _l2_buf = torch.empty(nbytes, dtype=torch.uint8, device=device or "cuda")
    _l2_buf.fill_(1)


def device_time_ms(fn: Callable[[], None], iters: int = 10, warmup: int = 3, flush: bool = False,
                   comm=None, reduce: str = "median") -> float:
    """Device time of ``fn`` in ms: per-iteration CUDA events, max over ranks of the
    median (or mean/min) over iterations."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        if flush:
            flush_l2()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if comm is not None and comm.Get_size() > 1:
            comm.Barrier()
        s.record()
        fn()
        e.record()
        e.synchronize()
        times.append(s.elapsed_time(e))
    val = {"median": statistics.median, "mean": statistics.fmean, "min": min}[reduce](times)
    return max_over_ranks(val, comm)


class ClockSampler:
    """Samples SM clocks / throttle reasons in the background during a timed region.

    In-process NVML (``pynvml``) when available: a query costs microseconds, so the samples really fall
    inside short timed regions and sampling does not disturb them.  The fallback spawns ``nvidia-smi``
    (tens of milliseconds of CPU and driver locks per query -- on an 8-rank job, eight of them at the
    moment the ranks enqueue their timed work were measured to skew the ranks against each other by
    ~100 us), so its first query is delayed."""

    QUERY = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int = 0, period_s: float = 0.2, first_delay_s: float = 0.0):
        self.gpu_index, self.period_s, self.first_delay_s = gpu_index, period_s, first_delay_s
        self.samples: list = []
        self.source = "none"
        self._stop = threading.Event()
        self._thread: Optional[threading.Thread] = None
        self._nvml = None
        try:
            import pynvml

            pynvml.nvmlInit()
            try:
                uuid = str(torch.cuda.get_device_properties(gpu_index).uuid)
                handle = pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid).encode())
            except Exception:
                handle = pynvml.nvmlDeviceGetHandleByIndex(gpu_index)
            self._nvml = (pynvml, handle)
            self.source = "nvml"
        except Exception:
            self._nvml = None

    def _sample_nvml(self):
        nv, h = self._nvml
        sm = nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)
        mx = nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)
        try:
            power = nv.nvmlDeviceGetPowerUsage(h) / 1000.0
        except Exception:
            power = 0.0
        try:
            mask = nv.nvmlDeviceGetCurrentClocksEventReasons(h)
        except Exception:
            mask = nv.nvmlDeviceGetCurrentClocksThrottleReasons(h)
        bits = (nv.nvmlClocksThrottleReasonHwSlowdown, nv.nvmlClocksThrottleReasonHwThermalSlowdown,
                nv.nvmlClocksThrottleReasonSwThermalSlowdown, nv.nvmlClocksThrottleReasonSwPowerCap)
        self.samples.append([str(sm), str(mx), f"{power:.1f}"] + ["Active" if mask & b else "Not Active" for b in bits])

    def _run(self):
        if self._nvml is None and self._stop.wait(max(self.first_delay_s, 0.05)):
            return
        if self._nvml is not None and self.first_delay_s > 0 and self._stop.wait(self.first_delay_s):
            return
        while not self._stop.is_set():
            try:
                if self._nvml is not None:
                    self._sample_nvml()
                else:
                    self.source = "nvidia-smi"
                    out = subprocess.run(
                        ["nvidia-smi", f"--query-gpu={self.QUERY}", "--format=csv,noheader,nounits",
                         "-i", str(self.gpu_index)], capture_output=True, text=True, timeout=5).stdout
                    parts = [p.strip() for p in out.strip().split(",")]
                    if len(parts) >= 7:
                        self.samples.append(parts)
            except Exception:
                pass
            self._stop.wait(self.period_s)

    def __enter__(self):
        self._thread = threading.Thread(target=self._run, daemon=True)
        self._thread.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        if self._thread:
            self._thread.join(timeout=10)

    def summary(self) -> dict:
        sm = [float(s[0]) for s in self.samples if s[0].replace(".", "").isdigit()]
        mx = [float(s[1]) for s in self.samples if s[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({n for s in self.samples for n, v in zip(names, s[3:7]) if v.lower() == "active"})
        return {
            "sm_mhz": statistics.median(sm) if sm else None,
            "sm_max_mhz": max(mx) if mx else None,
            "reasons": reasons,
            "samples": len(self.samples),
            "source": self.source,
        }
