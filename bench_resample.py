"""Benchmark of resampling (torchaudio.functional.resample as utils/audio.py:73 calls it, sinc_interp_hann, width 6, rolloff
0.99) on this library's polyphase kernel, against torchaudio on the host and on the same GPU.  Prints one JSON line.

    python bench_resample.py [--steps K] [--warmup W]

Workloads (seeded waveforms from oracle/resample_ref.py, output 44.1 kHz):
  api48, api16   B = 1, a 10 s clip at 48 kHz / 16 kHz: the reference audio of api.py:72
  b32            B = 32 x 10 s at 48 kHz: a corpus batch as preprocess.py:65 meets it
Arms:
  ours           the drop-in `resample` on CUDA tensors: `ms` is the median of K calls bracketed by CUDA events; `kernel_ms`
                 is the mean duration of `resample_kernel` in a separate torch.profiler run
  torchaudio_cpu_1t / _nt   torchaudio on the host with 1 thread (what preprocess.py sets) and with every usable thread (what
                 api.py runs): median host-clock time of max(3, K / 10) calls
  torchaudio_gpu torchaudio on CUDA tensors of the same GPU (its dense conv1d, cuDNN TF32 off), CUDA events after warm-up
For B = 1 the workload is also timed followed by the log-mel (this library's LogMelSpectrogram at the default MelConfig),
from the decoded host clip to the mel on the GPU, host clock around a synchronise: `chain_ours` resamples on the GPU,
`chain_torchaudio_cpu_nt` resamples on the host (all threads) and copies the result, as api.py does today.
`hbm_share` is the compulsory traffic (4 B per input and per output sample) over `kernel_ms`, as a share of the H100 SXM
data sheet's 3.35 TB/s: HBM bandwidth is the bound of this kernel, so this is how close it comes.  `max_abs_vs_fp64` compares
ours, and torchaudio's fp32 GPU output, with the float64 oracle on the timed inputs (every row for B = 1, three rows of the
batch).  The GPU's name, power limit and maximum SM clock are read in the same run.  Nothing is written to the tree."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit": q[1], "max_sm_clock": q[2]}
    except Exception as e:                                       # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({e})", "max_sm_clock": "unavailable"}


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def time_cuda(fn, steps, warmup):
    with torch.inference_mode():
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
    return median(ms)


def time_host(fn, reps, warmup=1):
    with torch.inference_mode():
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ms.append((time.perf_counter() - t0) * 1e3)
    return median(ms)


def kernel_ms(fn, reps):
    """mean device duration of resample_kernel over `reps` calls, from torch.profiler's CUDA activity"""
    from torch.profiler import ProfilerActivity, profile
    with torch.inference_mode(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    durs = [e.device_time for e in prof.events() if "resample_kernel" in e.name]
    return (sum(durs) / len(durs) / 1e3) if durs else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resample.py measures on a CUDA device; none is present")
    import torchaudio
    from oracle import mel_ref, resample_ref as R
    from stabletts_b200 import LogMelSpectrogram, resample
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    n_threads = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else os.cpu_count()
    mel = LogMelSpectrogram(**mel_ref.CONFIGS["default"]).to(dev)
    new = 44100
    result = {"bench": "resample", "method": "sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99", "new_freq": new,
              "host_threads": n_threads, "torchaudio": torchaudio.__version__, **gpu_info()}
    host_reps = max(3, args.steps // 10)
    for wname, orig, B in (("api48", 48000, 1), ("api16", 16000, 1), ("b32", 48000, 32)):
        L = 10 * orig
        kinds = ["speech", "noise", "sine", "square", "nyquist"]
        x_cpu = R.make_batch(["speech"] if B == 1 else [kinds[i % len(kinds)] for i in range(B)], 1000, L, orig)
        x = x_cpu.to(dev)
        n_out = R.out_length(orig, new, L)
        with torch.inference_mode():
            y = resample(x, orig, new)
            y_ta = torchaudio.functional.resample(x, orig, new)
        r = {"B": B, "orig_freq": orig, "L": L, "out_len": n_out}
        r["ours_ms"] = round(time_cuda(lambda: resample(x, orig, new), args.steps, args.warmup), 4)
        kms = kernel_ms(lambda: resample(x, orig, new), max(10, args.steps // 2))
        r["kernel_ms"] = None if kms is None else round(kms, 4)
        bytes_ = 4.0 * B * (L + n_out)
        r["compulsory_bytes"] = bytes_
        r["hbm_share"] = None if kms is None else round(bytes_ / HBM_BYTES_PER_S / (kms / 1e3), 4)
        r["audio_s_per_s"] = round(B * 10 / (r["ours_ms"] / 1e3), 1)
        r["torchaudio_gpu_ms"] = round(time_cuda(lambda: torchaudio.functional.resample(x, orig, new), args.steps,
                                                 args.warmup), 4)
        prev = torch.get_num_threads()
        for tag, nt in (("1t", 1), ("nt", n_threads)):
            torch.set_num_threads(nt)
            r[f"torchaudio_cpu_{tag}_ms"] = round(time_host(lambda: torchaudio.functional.resample(x_cpu, orig, new),
                                                            host_reps), 3)
        torch.set_num_threads(prev)
        r["speedup_vs_cpu_1t"] = round(r["torchaudio_cpu_1t_ms"] / r["ours_ms"], 1)
        r["speedup_vs_cpu_nt"] = round(r["torchaudio_cpu_nt_ms"] / r["ours_ms"], 1)
        r["speedup_vs_torchaudio_gpu"] = round(r["torchaudio_gpu_ms"] / r["ours_ms"], 2)
        rows = list(range(B)) if B == 1 else [0, 17, B - 1]
        ref = R.resample(x_cpu[rows], orig, new)
        r["max_abs_vs_fp64"] = float((y[rows].double().cpu() - ref).abs().max())
        r["torchaudio_fp32_max_abs_vs_fp64"] = float((y_ta[rows].double().cpu() - ref).abs().max())
        if B == 1:
            r["chain_ours_ms"] = round(time_host(lambda: mel(resample(x_cpu.to(dev), orig, new)), args.steps), 4)
            torch.set_num_threads(n_threads)
            r["chain_torchaudio_cpu_nt_ms"] = round(
                time_host(lambda: mel(torchaudio.functional.resample(x_cpu, orig, new).to(dev)), host_reps), 4)
            torch.set_num_threads(prev)
        result[wname] = r
    print(json.dumps(result))


if __name__ == "__main__":
    main()
