"""MRD forward + backward of real and fake audio (train.py:102 / :123) at B = 32, L = 20480: the library's
MultiResolutionDiscriminator against the staged reference module with torch's default TF32 convolutions and with TF32 off,
and train.py's discriminator and generator half-steps (no optimizer step) with only the MRD swapped and with generator, MPD,
MRD and mel loss all from the library.

    python bench_mrd.py [--iters 5 --runs 3 --batch 32 --length 20480 --steps 5]

Prints one JSON line.  The reference arms need oracle/_ref/vocos (staged by build() where a reference checkout exists) and
torchaudio; they read "not measured" when the staged copy (or torchaudio) is missing.  The card's name and power limit are
read in the same run.  Writes nothing."""
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


def gemm_flops(B, L, fft_sizes=(2048, 1024, 512)):
    """Forward + dgrad + wgrad FLOPs of band convs 1-4 for one waveform batch through every window (algorithmic)."""
    tot = 0.0
    for N in fft_sizes:
        T, F = L // (N // 4) + 1, N // 2 + 1
        for lo, hi in [(int(a * F), int(b * F)) for a, b in ((0, .1), (.1, .25), (.25, .5), (.5, .75), (.75, 1.0))]:
            W = hi - lo
            for i in range(1, 5):
                W = -(-W // 2) if i < 4 else W
                tot += 3 * 2.0 * B * T * W * 32 * 32 * (27 if i < 4 else 9)
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
    """train.py's D and G half-steps (forward, losses, backward; no optimizer step) in three arms, alternated step by step:
    "ours": the reference's generator, MPD and losses with the library's MRD; "ref_tf32": all reference (torch's default
    TF32 convolutions); "all_library": generator (Vocos in train mode), MPD, MRD and mel loss from the library, the
    scalar GAN losses the reference's.  Every arm starts from the same weights."""
    from oracle import stage_mel_loss
    from stabletts_b200 import MultiPeriodDiscriminator, MultiScaleMelSpectrogramLoss, Vocos
    ref_loss, ref_model, ref_disc, ref_cfg = stage_mel_loss.load_reference()
    torch.manual_seed(0)
    gen_r = ref_model.Vocos(ref_cfg.VocosConfig(), ref_cfg.MelConfig()).to(dev)
    mpd_r = ref_disc.MultiPeriodDiscriminator().to(dev)
    loss_r = ref_loss.MultiScaleMelSpectrogramLoss().to(dev)
    gen_o = Vocos().to(dev).train()
    gen_o.load_state_dict(gen_r.state_dict(), strict=True)
    mpd_o = MultiPeriodDiscriminator().to(dev)
    mpd_o.load_state_dict(mpd_r.state_dict(), strict=True)
    loss_o = MultiScaleMelSpectrogramLoss().to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    mels = torch.randn(B, 128, L // 512, device=dev, generator=g)
    with torch.no_grad():
        seg = gen_r(mels).shape[-1]
    audios = 0.1 * torch.randn(B, 1, seg, device=dev, generator=g)
    factor = ref_cfg.TrainConfig.mel_loss_factor

    def d_step(gen, mpd, mrd, mel_loss):
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
        return float(loss_s + loss_f)

    def g_step(gen, mpd, mrd, mel_loss):
        gen.zero_grad(set_to_none=True)
        fake = gen(mels).unsqueeze(1)
        loss_mel = mel_loss(audios, fake) * factor
        _, y_g, f_r, f_g = mpd(audios, fake)
        loss_f = ref_loss.feature_loss(f_r, f_g) + ref_loss.generator_loss(y_g)[0]
        _, y_g, f_r, f_g = mrd(audios, fake)
        loss_s = ref_loss.feature_loss(f_r, f_g) + ref_loss.generator_loss(y_g)[0]
        loss = loss_s + loss_f + loss_mel
        loss.backward()
        return float(loss)

    arms = {"ours": (gen_r, mpd_r, ours, loss_r), "ref_tf32": (gen_r, mpd_r, ref, loss_r),
            "all_library": (gen_o, mpd_o, ours, loss_o)}
    out = {"segment": seg}
    for name, fn in (("d", d_step), ("g", g_step)):
        losses = {k: fn(*mods) for k, mods in arms.items()}
        out[f"{name}_loss_rel_vs_ref_tf32"] = {k: abs(v - losses["ref_tf32"]) / abs(losses["ref_tf32"])
                                               for k, v in losses.items() if k != "ref_tf32"}
        ts = {k: [] for k in arms}
        for _ in range(steps):
            for k, mods in arms.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                fn(*mods)
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
    from stabletts_b200 import MultiResolutionDiscriminator
    dev = torch.device("cuda:0")
    name, limit = card()
    B, L = args.batch, args.length
    res = {"bench": "mrd", "card": name, "power_limit": limit, "B": B, "L": L}
    torch.manual_seed(0)
    ours = MultiResolutionDiscriminator().to(dev)
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
        ref = disc.MultiResolutionDiscriminator().to(dev)
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
