"""The Vocos generator's training step on the GPU against the reference module.  Prints one JSON line.

    python bench_vocos_train.py [--iters 5] [--warmup 2] [--runs 3] [--batch 32] [--frames 40] [--steps 5]

Generator forward + backward at B = 32, T = 40 mel frames (TrainConfig's batch and 20480-sample segment), the vocos
training config 768 / 2048 / 12: stabletts_b200's ``Vocos`` against the reference's (the staged oracle/_ref/vocos copy)
with the same weights, the reference with torch's default TF32 settings (TF32 convolutions, fp32 matmuls) and with TF32 off
everywhere; the arms alternate and each time is the median of `--runs` runs of `--iters` calls timed with CUDA events.
Parity: the largest L2-relative error over the parameter gradients of the drop-in against each reference arm.  "profile":
one separate forward + backward with the library's per-launch CUDA-event profiling (st_profile_*): the GEMM launches'
summed time and count against the rest of the call (row kernels, transposes, splits).  "resync_ms": the extra time of a
forward + backward right after every parameter changed (an optimizer step): st_load_weight of every tensor, finalize and
the transposed packs of the first backward.  "half_step": train.py's generator half-step (:113-128: mel loss, MPD and MRD
feature and generator losses, backward) with Vocos, MPD and the mel loss from the library (the MRD stays the reference's)
against all-reference, arms alternated, medians of `--steps`.  "not measured" where the staged copy (or torchaudio) is
missing.  The card's name and power limit are read in the same run.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_mpd import card, cuda_ms  # noqa: E402


def set_tf32(on: bool):
    torch.backends.cudnn.allow_tf32 = on                  # torch's default: TF32 convolutions, fp32 matmuls
    torch.backends.cuda.matmul.allow_tf32 = False


def grads(m):
    return [p.grad.detach().clone() for p in m.parameters()]


def profile(ours, fn):
    import ctypes as C
    from stabletts_b200 import _lib
    lib = _lib.load_library()
    n = _lib.ST_PROF_NCAT
    fn()
    torch.cuda.synchronize()
    lib.st_profile_begin(ours._handle)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    fn()
    t1.record()
    torch.cuda.synchronize()
    a, f, b, k = (C.c_double * n)(), (C.c_double * n)(), (C.c_double * n)(), (C.c_int64 * n)()
    lib.st_profile_end(ours._handle, a, f, b, k)
    gemm = [i for i, nm in enumerate(_lib.ST_PROF_NAMES) if nm.startswith("gemm")]
    ms = sum(a[i] for i in gemm)
    fl = sum(f[i] for i in gemm)
    total = t0.elapsed_time(t1)
    return {"call_ms_profiled": round(total, 3), "gemm_ms": round(ms, 3), "gemm_launches": int(sum(k[i] for i in gemm)),
            "gemm_tflops": round(fl / (ms * 1e-3) / 1e12, 2) if ms else None, "rest_of_call_ms": round(total - ms, 3)}


def half_step(ours, ref, mels, steps, dev):
    """train.py's generator half-step; arm "ours": library Vocos, MPD and mel loss; arm "ref": all reference"""
    from oracle import stage_mel_loss
    from stabletts_b200 import MultiPeriodDiscriminator, MultiScaleMelSpectrogramLoss
    ref_loss, _, ref_disc, ref_cfg = stage_mel_loss.load_reference()
    torch.manual_seed(1)
    mpd_r = ref_disc.MultiPeriodDiscriminator().to(dev)
    mrd = ref_disc.MultiResolutionDiscriminator().to(dev)
    mpd_o = MultiPeriodDiscriminator().to(dev)
    mpd_o.load_state_dict(mpd_r.state_dict(), strict=True)
    loss_r = ref_loss.MultiScaleMelSpectrogramLoss().to(dev)
    loss_o = MultiScaleMelSpectrogramLoss().to(dev)
    g = torch.Generator(device=dev).manual_seed(2)
    audios = 0.1 * torch.randn(mels.shape[0], 1, mels.shape[2] * 512, device=dev, generator=g)
    factor = ref_cfg.TrainConfig.mel_loss_factor

    def step(gen, mpd, mel_loss):
        gen.zero_grad(set_to_none=True)
        fake = gen(mels).unsqueeze(1)
        loss_mel = mel_loss(audios, fake) * factor
        _, y_g, f_r, f_g = mpd(audios, fake)
        loss_f = ref_loss.feature_loss(f_r, f_g) + ref_loss.generator_loss(y_g)[0]
        _, y_g, f_r, f_g = mrd(audios, fake)
        loss_s = ref_loss.feature_loss(f_r, f_g) + ref_loss.generator_loss(y_g)[0]
        (loss_s + loss_f + loss_mel).backward()

    arms = {"ours": lambda: step(ours, mpd_o, loss_o), "ref_tf32": lambda: step(ref, mpd_r, loss_r)}
    for f in arms.values():
        f()
    ts = {k: [] for k in arms}
    for _ in range(steps):
        for k, f in arms.items():
            ts[k].append(cuda_ms(f, 1))
    out = {f"{k}_ms": round(statistics.median(v), 2) for k, v in ts.items()}
    out["speedup_vs_ref_tf32"] = round(statistics.median(ts["ref_tf32"]) / statistics.median(ts["ours"]), 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    from stabletts_b200 import Vocos
    dev = torch.device("cuda:0")
    name, limit = card()
    B, T = args.batch, args.frames
    res = {"bench": "vocos_train", "card": name, "power_limit": limit, "B": B, "T": T, "dims": "768/2048/12"}
    torch.manual_seed(0)
    ours = Vocos().to(dev).train()
    g = torch.Generator(device=dev).manual_seed(1)
    mels = torch.randn(B, 128, T, device=dev, generator=g)
    up = torch.randn(B, T * 512, device=dev, generator=g)

    def step(m):
        m.zero_grad(set_to_none=True)
        (m(mels) * up).sum().backward()

    arms = {"ours": lambda: step(ours)}
    ref = None
    try:
        from oracle import stage_mel_loss
        _, ref_model, _, ref_cfg = stage_mel_loss.load_reference()
        ref = ref_model.Vocos(ref_cfg.VocosConfig(), ref_cfg.MelConfig()).to(dev).train()
        ref.load_state_dict(ours.state_dict(), strict=True)
    except Exception as e:                                   # noqa: BLE001
        res["reference"] = f"not measured ({e})"

    def ref_arm(tf32):
        def run():
            set_tf32(tf32)
            try:
                step(ref)
            finally:
                set_tf32(True)
        return run

    if ref is not None:
        arms["ref_tf32"] = ref_arm(True)
        arms["ref_fp32"] = ref_arm(False)
    got = {}
    for k, f in arms.items():
        f()
        got[k] = grads(ours if k == "ours" else ref)
    for _ in range(args.warmup - 1):
        for f in arms.values():
            f()
    times = {k: [] for k in arms}
    for _ in range(args.runs):
        for k, f in arms.items():
            times[k].append(cuda_ms(f, args.iters))
    med = {k: statistics.median(v) for k, v in times.items()}
    res["ours_ms"] = round(med["ours"], 3)
    res["ours_runs_ms"] = [round(t, 3) for t in times["ours"]]
    for k in ("ref_tf32", "ref_fp32"):
        if k in med:
            res[k + "_ms"] = round(med[k], 3)
            res[k + "_runs_ms"] = [round(t, 3) for t in times[k]]
            res["speedup_vs_" + k] = round(med[k] / med["ours"], 3)
            res["grad_parity_max_l2rel_vs_" + k] = max(float((a - b).norm() / b.norm()) for a, b in zip(got["ours"], got[k]))
    res["profile"] = profile(ours, lambda: step(ours))
    resync = []
    for _ in range(args.runs):
        with torch.no_grad():
            for p in ours.parameters():
                p.mul_(1.0)                                  # bumps every version counter, as an optimizer step does
        t_changed = cuda_ms(lambda: step(ours), 1)
        resync.append(t_changed - cuda_ms(lambda: step(ours), 1))
    res["resync_ms"] = round(statistics.median(resync), 3)
    if ref is not None:
        try:
            res["half_step"] = half_step(ours, ref, mels, args.steps, dev)
        except Exception as e:                               # noqa: BLE001
            res["half_step"] = f"not measured ({e})"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
