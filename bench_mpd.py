"""The Vocos trainer's multi-period discriminator on the GPU against the reference module.  Prints one JSON line.

    python bench_mpd.py [--iters 5] [--warmup 2] [--batch 32] [--length 20480]

MPD forward + backward at B = 32, L = 20480 (TrainConfig's batch and segment), as train.py's generator half-step runs it:
real and generated audio, parameters requiring grad, gradients into y_hat, a loss on every score and fmap.
stabletts_b200's ``MultiPeriodDiscriminator`` against the reference's (the staged oracle/_ref/vocos copy) with the same
weights, the reference with its default TF32 convolutions and with TF32 off; the arms alternate and each time is the median
of `--runs` runs of `--iters` calls timed with CUDA events.  Parity: the largest max-rel over every score of the drop-in
against each reference arm.  "whole_call_gemm_tflops": the algorithmic FLOPs of convs 1-4 (forward, input and weight
gradients, counted from the shapes without the packings' zero lanes) over the drop-in's whole call time.  "profile": one
separate call with the library's per-launch CUDA-event profiling (st_profile_*): the summed time and count of the GEMM
launches and the FLOPs the engine counts for them (the packings' zero lanes included), so their per-launch rate, and the
time of every other launch (row kernels, packing) as the rest of the call.
Then train.py's discriminator half-step (:95-110) and generator half-step (:113-128, mel loss included) with the reference's
Vocos 768 / 2048 / 12, MRD and losses, with only the MPD swapped, arms alternated from the same seed, medians of `--steps`.
"not measured" when the staged copy (or torchaudio) is missing.  The card's name and power limit are read in the same run.
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except Exception as e:                                   # noqa: BLE001
        limit = f"unknown ({e})"
    return name, limit


def cuda_ms(fn, iters):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def gemm_flops(B, L, periods=(2, 3, 5, 7, 11)):
    """Forward + dgrad + wgrad FLOPs of convs 1-4 for one waveform batch through every period (algorithmic: 5 taps)."""
    chans = (1, 32, 128, 512, 1024, 1024)
    tot = 0.0
    for p in periods:
        H = -(-L // p)
        for i in range(5):
            H = -(-H // 3) if i < 4 else H
            if i >= 1:
                tot += 3 * 2.0 * B * p * H * chans[i] * chans[i + 1] * 5
    return tot


def profile(ours, fn):
    """GEMM launches vs everything else in one call, from the library's per-launch event profiling."""
    import ctypes as C
    from stabletts_b200 import _lib
    lib = _lib.load_library()
    n = _lib.ST_PROF_NCAT
    torch.cuda.synchronize()
    for d in ours.discriminators:
        lib.st_profile_begin(d._handle)
    t0 = torch.cuda.Event(enable_timing=True)
    t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    fn()
    t1.record()
    torch.cuda.synchronize()
    ms = flops = 0.0
    launches = 0
    for d in ours.discriminators:
        a, f, b, k = (C.c_double * n)(), (C.c_double * n)(), (C.c_double * n)(), (C.c_int64 * n)()
        lib.st_profile_end(d._handle, a, f, b, k)
        ms += a[0]
        flops += f[0]
        launches += k[0]
    total = t0.elapsed_time(t1)
    return {"call_ms_profiled": round(total, 3), "gemm_ms": round(ms, 3), "gemm_launches": int(launches),
            "gemm_engine_tflops": round(flops / (ms * 1e-3) / 1e12, 2) if ms else None,
            "rest_of_call_ms": round(total - ms, 3)}


def half_steps(ours, ref, B, L, steps, dev):
    """train.py's D and G half-steps with the reference's generator, MRD and losses; only the MPD differs."""
    from oracle import stage_mel_loss
    ref_loss, ref_model, ref_disc, ref_cfg = stage_mel_loss.load_reference()
    torch.manual_seed(0)
    gen = ref_model.Vocos(ref_cfg.VocosConfig(), ref_cfg.MelConfig()).to(dev)
    mrd = ref_disc.MultiResolutionDiscriminator().to(dev)
    mel_loss = ref_loss.MultiScaleMelSpectrogramLoss().to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    mels = torch.randn(B, 128, L // 512, device=dev, generator=g)
    with torch.no_grad():
        seg = gen(mels).shape[-1]
    audios = 0.1 * torch.randn(B, 1, seg, device=dev, generator=g)
    factor = ref_cfg.TrainConfig.mel_loss_factor

    def d_step(mpd):
        mpd.zero_grad(set_to_none=True)
        mrd.zero_grad(set_to_none=True)
        with torch.no_grad():
            fake = gen(mels).unsqueeze(1)
        y_r, y_g, _, _ = mpd(audios, fake.detach())
        loss_f, _, _ = ref_loss.discriminator_loss(y_r, y_g)
        y_r, y_g, _, _ = mrd(audios, fake.detach())
        loss_s, _, _ = ref_loss.discriminator_loss(y_r, y_g)
        (loss_s + loss_f).backward()
        torch.nn.utils.clip_grad_norm_(mpd.parameters(), 1000)
        torch.nn.utils.clip_grad_norm_(mrd.parameters(), 1000)

    def g_step(mpd):
        gen.zero_grad(set_to_none=True)
        fake = gen(mels).unsqueeze(1)
        loss_mel = mel_loss(audios, fake) * factor
        _, y_g, f_r, f_g = mpd(audios, fake)
        loss_f = ref_loss.feature_loss(f_r, f_g) + ref_loss.generator_loss(y_g)[0]
        _, y_g, f_r, f_g = mrd(audios, fake)
        loss_s = ref_loss.feature_loss(f_r, f_g) + ref_loss.generator_loss(y_g)[0]
        (loss_s + loss_f + loss_mel).backward()

    out = {"segment": seg}
    for name, fn in (("d", d_step), ("g", g_step)):
        for m in (ours, ref):
            fn(m)
        ts = {"ours": [], "ref_tf32": []}
        for _ in range(steps):
            for k, m in (("ours", ours), ("ref_tf32", ref)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                fn(m)
                b.record()
                torch.cuda.synchronize()
                ts[k].append(a.elapsed_time(b))
        for k, v in ts.items():
            out[f"{name}_{k}_ms"] = round(statistics.median(v), 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--length", type=int, default=20480)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    from stabletts_b200 import MultiPeriodDiscriminator
    dev = torch.device("cuda:0")
    name, limit = card()
    B, L = args.batch, args.length
    res = {"bench": "mpd", "card": name, "power_limit": limit, "B": B, "L": L}
    torch.manual_seed(0)
    ours = MultiPeriodDiscriminator().to(dev)
    y = 0.3 * torch.randn(B, 1, L, device=dev)
    y_hat = (0.3 * torch.randn(B, 1, L, device=dev)).requires_grad_(True)

    def step(m):
        y_d_rs, y_d_gs, fmap_rs, fmap_gs = m(y, y_hat)
        loss = sum(s.mean() for s in y_d_rs + y_d_gs) + sum(f.mean() for fs in fmap_rs + fmap_gs for f in fs)
        loss.backward()
        return y_d_rs + y_d_gs

    arms = {"ours": lambda: step(ours)}
    ref = None
    try:
        from oracle import stage_mel_loss
        _, _, disc, _ = stage_mel_loss.load_reference()
        ref = disc.MultiPeriodDiscriminator().to(dev)
        ref.load_state_dict(ours.state_dict(), strict=True)
    except Exception as e:                                   # noqa: BLE001
        res["reference"] = f"not measured ({e})"

    def ref_arm(tf32):
        def run():
            torch.backends.cudnn.allow_tf32 = tf32
            try:
                return step(ref)
            finally:
                torch.backends.cudnn.allow_tf32 = True
        return run

    if ref is not None:
        arms["ref_tf32"] = ref_arm(True)
        arms["ref_fp32"] = ref_arm(False)
    scores = {k: [s.detach().clone() for s in f()] for k, f in arms.items()}
    for _ in range(args.warmup - 1):
        for f in arms.values():
            f()
    times = {k: [] for k in arms}
    launches0 = sum(d.launch_count() for d in ours.discriminators)
    for _ in range(args.runs):
        for k, f in arms.items():
            times[k].append(cuda_ms(f, args.iters))
    launches = (sum(d.launch_count() for d in ours.discriminators) - launches0) / (args.runs * args.iters)
    med = {k: statistics.median(v) for k, v in times.items()}
    res["ours_ms"] = round(med["ours"], 3)
    res["ours_runs_ms"] = [round(t, 3) for t in times["ours"]]
    res["launches_per_call"] = launches
    res["whole_call_gemm_tflops"] = round(2 * gemm_flops(B, L) / (med["ours"] * 1e-3) / 1e12, 2)    # real + fake
    res["profile"] = profile(ours, lambda: step(ours))
    for k in ("ref_tf32", "ref_fp32"):
        if k in med:
            res[k + "_ms"] = round(med[k], 3)
            res[k + "_runs_ms"] = [round(t, 3) for t in times[k]]
            res["speedup_vs_" + k] = round(med[k] / med["ours"], 3)
            res["parity_max_rel_vs_" + k] = max(float((a - b).abs().max() / b.abs().max()) for a, b in zip(scores["ours"], scores[k]))
    if ref is not None:
        res["half_steps"] = half_steps(ours, ref, B, L, args.steps, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
