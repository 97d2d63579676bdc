"""Benchmark of log-mel extraction (utils/audio.py::LogMelSpectrogram at the default MelConfig) on this library's fp32 FFT
kernel, against the reference's own module on the same GPU (torch.stft on cuFFT, then MelScale and the log).  Prints one
JSON line.

    python bench_mel.py [--steps K] [--warmup W]

Workloads (seeded waveforms from oracle/mel_ref.py, 44.1 kHz, n_fft 2048, hop 512, 128 mels):
  api   B = 1, 10 s (861 frames): the reference clip api.py turns into a mel
  b32   B = 32 x 10 s: a preprocess.py-style batch
Per workload: `ms` is the median of K module calls, each bracketed by CUDA events; `kernel_ms` is the mean duration of
`mel_kernel` in a separate torch.profiler run; frames/s and audio-seconds/s are over `ms`.  `compulsory_bytes_bound` is the
least time the HBM could take to read 4 B per input sample and write 4 * n_mels B per output frame at the H100 SXM data
sheet's 3.35 TB/s, over `kernel_ms`: a bandwidth bound, not a measured bandwidth.  The reference arm is the staged
reference module (oracle/_ref, made by build() where a checkout exists), TF32 off; `max_abs_vs_reference` compares the two
arms' fp32 outputs and `max_abs_vs_fp64` compares ours with the float64 oracle (api workload).  The GPU's name, power limit
and maximum SM clock are read in the same run.  Nothing is written to the tree."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

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


def time_calls(fn, x, steps, warmup):
    with torch.inference_mode():
        for _ in range(warmup):
            fn(x)
        torch.cuda.synchronize()
        ms = []
        for _ in range(steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(x)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
    return median(ms)


def kernel_ms(fn, x, reps):
    """mean device duration of mel_kernel over `reps` calls, from torch.profiler's CUDA activity"""
    from torch.profiler import ProfilerActivity, profile
    with torch.inference_mode(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn(x)
        torch.cuda.synchronize()
    durs = [e.device_time for e in prof.events() if "mel_kernel" in e.name]
    return (sum(durs) / len(durs) / 1e3) if durs else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mel.py measures on a CUDA device; none is present")
    from oracle import mel_ref as M, stage_mel
    from stabletts_b200 import LogMelSpectrogram
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    cfg = M.CONFIGS["default"]
    ours = LogMelSpectrogram(**cfg).to(dev)
    ref = None
    if stage_mel.available():
        ref = stage_mel.load_reference()(**cfg).to(dev)
        ref.load_state_dict(ours.state_dict())                  # the same window and fb in both arms
    result = {"bench": "log_mel", "config": "MelConfig() (44.1 kHz, n_fft 2048, hop 512, 128 mels)",
              "reference_kind": "reference" if ref is not None else "absent", **gpu_info()}
    sr = cfg["sample_rate"]
    L = 10 * sr
    kinds = ["speech", "noise", "lowpass", "sine", "square", "quiet"]
    for wname, B in (("api", 1), ("b32", 32)):
        x = M.make_batch(["speech"] if B == 1 else [kinds[i % len(kinds)] for i in range(B)], 401, L, sr).to(dev)
        T = M.n_frames(cfg, L)
        with torch.inference_mode():
            y = ours(x)
        ms = time_calls(ours, x, args.steps, args.warmup)
        kms = kernel_ms(ours, x, max(10, args.steps // 2))
        bytes_ = 4.0 * B * L + 4.0 * cfg["n_mels"] * B * T
        r = {"B": B, "L": L, "frames": B * T, "ms": round(ms, 4), "kernel_ms": None if kms is None else round(kms, 4),
             "frames_per_s": round(B * T / (ms / 1e3), 1), "audio_s_per_s": round(B * L / sr / (ms / 1e3), 1),
             "compulsory_bytes": bytes_,
             "compulsory_bytes_bound": None if kms is None else round(bytes_ / HBM_BYTES_PER_S / (kms / 1e3), 4)}
        if ref is not None:
            r["reference_ms"] = round(time_calls(ref, x, args.steps, args.warmup), 4)
            r["speedup"] = round(r["reference_ms"] / ms, 3)
            with torch.inference_mode():
                r["max_abs_vs_reference"] = float((ref(x) - y).abs().max())
        if B == 1:
            r["max_abs_vs_fp64"] = float((y.double().cpu() - M.log_mel(x.cpu(), torch.hann_window(cfg["n_fft"]),
                                                                        ours.mel_scale.fb.cpu(), cfg)).abs().max())
        result[wname] = r
    print(json.dumps(result))


if __name__ == "__main__":
    main()
