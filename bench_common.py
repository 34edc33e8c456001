"""Shared measurement plumbing of bench.py and its workload modules (bench_wavernn / bench_tacotron / bench_e2e).

  Ctx           rank / world / device, torch.distributed set-up (NCCL; env untouched), barrier
  Ctx.timed     W warm-up steps -> K timed steps ("burst": clocks as they come) -> >= soak_s seconds of the same step ->
                K timed steps ("soaked": the steady state a long job sees).  CUDA events on the launching stream
                bracketed by barrier + synchronize, max over ranks.  `value` everywhere is the SOAKED figure.
  ClockSampler  NVML SM clock / throttle reasons sampled every ~10 ms on a thread; statistics over a time window
  cpu_child     CPU baseline in a child process with CUDA hidden and a hard time limit
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent


def log(msg: str) -> None:
    print(f"[bench {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def host_threads() -> int:
    """CPU threads this job may really use: affinity mask capped by the cgroup CPU quota (a container
    on a 200-core host with an 8-core quota must not spawn 200 spinning OpenMP threads)."""
    n = len(os.sched_getaffinity(0))
    try:
        txt = Path("/sys/fs/cgroup/cpu.max").read_text().split()
        if txt[0] != "max":
            n = min(n, max(1, int(float(txt[0]) / float(txt[1]) + 0.5)))
    except Exception:
        try:
            q = int(Path("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read_text())
            per = int(Path("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read_text())
            if q > 0:
                n = min(n, max(1, int(q / per + 0.5)))
        except Exception:
            pass
    return max(1, min(n, 64))


def cpu_child(workload: str, amount: int, threads: int, timeout: float):
    """Run the CPU baseline in a child process with CUDA hidden (SURVEY.md fact 11) and a hard
    time limit; returns the child's JSON dict or None."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS=str(threads), MKL_NUM_THREADS=str(threads))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    try:
        out = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--cpu-child", workload, str(amount), str(threads)],
                             env=env, capture_output=True, text=True, timeout=timeout)
        for line in reversed(out.stdout.strip().splitlines()):
            if line.startswith("{"):
                return json.loads(line)
        log(f"cpu child produced no result: {out.stderr[-500:]}")
    except subprocess.TimeoutExpired:
        log(f"cpu child exceeded {timeout}s")
    return None


def peaks():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.is_file():
        d = json.loads(p.read_text())
        return {"hbm_gbs": d["hbm_gbs"], "tflops_burst": d["bf16_tflops"],
                "tflops_sustained": d.get("bf16_tflops_sustained", d["bf16_tflops"]), "source": "measured (MEASURED_PEAKS.json)"}
    return {"hbm_gbs": 3350.0, "tflops_burst": 989.0, "tflops_sustained": 989.0, "source": "H100 SXM data sheet (700 W), not measured"}


class ClockSampler:
    """SM clock and throttle reasons of one GPU, sampled on a thread through NVML (nvidia_ml_py) every ~10 ms with a
    wall-clock stamp; `window(t0, t1)` summarises the samples taken inside [t0, t1] (time.perf_counter)."""

    REASONS = ((0x8, "hw_slowdown"), (0x40, "hw_thermal_slowdown"), (0x20, "sw_thermal_slowdown"), (0x4, "sw_power_cap"))

    def __init__(self, index: int):
        self.index = index
        self.samples = []  # (t, sm_mhz, reasons_mask, power_w)
        self._stop = threading.Event()
        self._thread = None
        self._h = None
        self.sm_max = None
        self.err = None
        try:
            import pynvml

            self._nv = pynvml
            pynvml.nvmlInit()
            try:
                import torch

                uuid = str(torch.cuda.get_device_properties(index).uuid)
                if not uuid.startswith("GPU-"):
                    uuid = "GPU-" + uuid
                self._h = pynvml.nvmlDeviceGetHandleByUUID(uuid.encode() if hasattr(uuid, "encode") else uuid)
            except Exception:
                self._h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.sm_max = float(pynvml.nvmlDeviceGetMaxClockInfo(self._h, pynvml.NVML_CLOCK_SM))
        except Exception as e:  # pragma: no cover
            self.err = f"NVML unavailable: {e}"

    def start(self):
        if self._h is None:
            return self
        self._thread = threading.Thread(target=self._run, daemon=True)
        self._thread.start()
        return self

    def _run(self):
        nv = self._nv
        reasons_fn = getattr(nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or nv.nvmlDeviceGetCurrentClocksThrottleReasons
        while not self._stop.is_set():
            try:
                sm = float(nv.nvmlDeviceGetClockInfo(self._h, nv.NVML_CLOCK_SM))
                rs = int(reasons_fn(self._h))
                try:
                    pw = nv.nvmlDeviceGetPowerUsage(self._h) / 1000.0
                except Exception:
                    pw = None
                self.samples.append((time.perf_counter(), sm, rs, pw))
            except Exception as e:  # pragma: no cover
                self.err = str(e)
                break
            time.sleep(0.008)

    def stop(self):
        self._stop.set()
        if self._thread is not None:
            self._thread.join(timeout=1.0)

    def window(self, t0: float, t1: float):
        if self._h is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [self.err or "NVML unavailable"], "samples": 0}
        rows = [s for s in self.samples if t0 <= s[0] <= t1]
        sm = sorted(s[1] for s in rows)
        mask = 0
        for s in rows:
            mask |= s[2]
        counts = {name: sum(1 for s in rows if s[2] & bit) for bit, name in self.REASONS}
        pw = [s[3] for s in rows if s[3] is not None]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_min_mhz": sm[0] if sm else None, "sm_max_mhz": self.sm_max,
                "reasons": [name for bit, name in self.REASONS if mask & bit], "reason_samples": {k: v for k, v in counts.items() if v},
                "power_w_max": max(pw) if pw else None, "samples": len(rows), "window_s": round(t1 - t0, 4)}


class Ctx:
    """one process per GPU (torchrun env: RANK / LOCAL_RANK / WORLD_SIZE / MASTER_*), NCCL for the plumbing"""

    def __init__(self):
        import torch
        import torch.distributed as dist

        self.torch, self.dist = torch, dist
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(self.local)
        self.dev = torch.device("cuda", self.local)
        if self.world > 1 and not dist.is_initialized():
            dist.init_process_group("nccl", device_id=self.dev)
        self.sampler = ClockSampler(self.local).start()
        self.outputs = {}  # name -> what the last resident (timed) step returned; bench.py --dump-outputs writes it

    def close(self):
        self.sampler.stop()
        if self.world > 1 and self.dist.is_initialized():
            self.dist.destroy_process_group()

    def barrier(self):
        self.torch.cuda.synchronize()
        if self.world > 1:
            self.dist.barrier()
        self.torch.cuda.synchronize()

    def _region(self, fn, k, host_clock: bool):
        """K calls bracketed by barrier + synchronize; device time (CUDA events on the current stream) - or the host
        wall clock when the step contains host work the events cannot see - max over ranks.  Returns (ms, t0, t1)."""
        torch = self.torch
        self.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        for _ in range(k):
            fn()
        e1.record()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        ms = e0.elapsed_time(e1)
        if host_clock:
            ms = max(ms, (t1 - t0) * 1e3)
        t = torch.tensor([ms], device=self.dev)
        if self.world > 1:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        self.barrier()
        return float(t.item()), t0, t1

    def timed(self, fn, k: int, warmup: int, soak_s: float = 2.0, host_clock: bool = False):
        """see module docstring.  Returns {"ms": soaked total, "ms_burst": ..., "clocks": ..., "clocks_burst": ...}"""
        for _ in range(max(0, warmup)):
            fn()
        ms_b, b0, b1 = self._region(fn, k, host_clock)
        t_end = time.perf_counter() + soak_s
        n_soak = 0
        while time.perf_counter() < t_end:
            fn()
            n_soak += 1
            if n_soak % 8 == 0:
                self.torch.cuda.synchronize()
        ms_s, s0, s1 = self._region(fn, k, host_clock)
        return {"ms": ms_s, "ms_burst": ms_b, "soak_steps": n_soak, "soak_s": soak_s,
                "clocks": self.sampler.window(s0, s1), "clocks_burst": self.sampler.window(b0, b1),
                "clocks_soak": self.sampler.window(b1, s0)}
