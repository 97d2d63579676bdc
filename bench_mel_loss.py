"""The Vocos trainer's multi-scale mel loss on the GPU against the reference module.  Prints one JSON line.

    python bench_mel_loss.py [--iters 20] [--warmup 3] [--steps 6]

- (a) loss forward + backward (d loss / d y) at B = 32, L = 20480 (TrainConfig's batch and segment): stabletts_b200's
  ``MultiScaleMelSpectrogramLoss`` against the reference's (the staged oracle/_ref/vocos copy) on the same CUDA tensors,
  timed with CUDA events after a warm-up.
- (b) the reference's own generator half-step (vocoders/vocos/train.py:113-128: Vocos 768 / 2048 / 12 on a (B, 128, 40)
  mel, MPD + MRD, the mel loss x 15, feature and generator losses, backward), with each loss, alternated from the same
  seed; the two mel-loss values must agree within the test bar (1e-6 relative).
"not measured" when the staged copy (or torchaudio) is missing.  The card's name and power limit are read in the same run.
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
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


def cuda_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--batch", type=int, default=32)
    args = ap.parse_args()
    from stabletts_b200 import MultiScaleMelSpectrogramLoss
    dev = torch.device("cuda:0")
    name, limit = card()
    res = {"metric": "mel_loss", "gpu": name, "power_limit": limit, "B": args.batch, "L": 20480}
    B, L = args.batch, 20480
    g = torch.Generator(device=dev).manual_seed(0)
    x = 0.1 * torch.randn(B, 1, L, device=dev, generator=g)
    y0 = x + 0.02 * torch.randn(B, 1, L, device=dev, generator=g)
    ours = MultiScaleMelSpectrogramLoss().to(dev)
    try:
        from oracle import stage_mel_loss
        ref_loss, ref_model, ref_disc, ref_cfg = stage_mel_loss.load_reference()
        ref = ref_loss.MultiScaleMelSpectrogramLoss().to(dev)
        ours.load_state_dict(ref.state_dict(), strict=True)
    except Exception as e:                                   # noqa: BLE001
        ref = None
        res["reference"] = f"not measured ({type(e).__name__}: {e})"

    def step(m):
        def run():
            y = y0.clone().requires_grad_()
            m(x, y).backward()
            return y.grad
        return run

    res["a_ours_ms"] = round(cuda_ms(step(ours), args.iters, args.warmup), 3)
    launches = ours.launch_count()
    step(ours)()
    res["a_ours_launches"] = ours.launch_count() - launches
    if ref is not None:
        res["a_reference_ms"] = round(cuda_ms(step(ref), args.iters, args.warmup), 3)
        res["a_speedup"] = round(res["a_reference_ms"] / res["a_ours_ms"], 2)
        with torch.no_grad():
            lo, lr = float(ours(x, y0)), float(ref(x, y0))
        res["a_loss_rel_diff"] = abs(lo - lr) / abs(lr)
        gy_o, gy_r = step(ours)(), step(ref)()
        res["a_grad_l2_rel_diff"] = float((gy_o - gy_r).norm() / gy_r.norm())

        # (b) the generator half-step of train.py:113-128 with each mel loss, alternated from the same seed
        torch.manual_seed(0)
        gen = ref_model.Vocos(ref_cfg.VocosConfig(), ref_cfg.MelConfig()).to(dev)
        mpd, mrd = ref_disc.MultiPeriodDiscriminator().to(dev), ref_disc.MultiResolutionDiscriminator().to(dev)
        mels = torch.randn(B, 128, L // 512, device=dev, generator=g)
        with torch.no_grad():
            seg = gen(mels).shape[-1]
        audios = 0.1 * torch.randn(B, 1, seg, device=dev, generator=g)
        factor = ref_cfg.TrainConfig.mel_loss_factor

        def half_step(loss_fn, out):
            gen.zero_grad(set_to_none=True)
            audios_fake = gen(mels).unsqueeze(1)
            loss_mel = loss_fn(audios, audios_fake) * factor
            _, y_df_hat_g, fmap_f_r, fmap_f_g = mpd(audios, audios_fake)
            loss_fm_f = ref_loss.feature_loss(fmap_f_r, fmap_f_g)
            loss_gen_f, _ = ref_loss.generator_loss(y_df_hat_g)
            _, y_ds_hat_g, fmap_s_r, fmap_s_g = mrd(audios, audios_fake)
            loss_fm_s = ref_loss.feature_loss(fmap_s_r, fmap_s_g)
            loss_gen_s, _ = ref_loss.generator_loss(y_ds_hat_g)
            (loss_gen_s + loss_gen_f + loss_fm_s + loss_fm_f + loss_mel).backward()
            out.append(loss_mel.detach())

        mel_o, mel_r, t_o, t_r = [], [], [], []
        for arm, lst in ((ours, mel_o), (ref, mel_r)):        # warm-up of both arms
            half_step(arm, lst)
        torch.cuda.synchronize()
        for _ in range(args.steps):
            for arm, lst, ts in ((ours, mel_o, t_o), (ref, mel_r, t_r)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                half_step(arm, lst)
                b.record()
                torch.cuda.synchronize()
                ts.append(a.elapsed_time(b))
        res["b_segment"] = seg
        res["b_ours_ms"] = round(sorted(t_o)[len(t_o) // 2], 2)
        res["b_reference_ms"] = round(sorted(t_r)[len(t_r) // 2], 2)
        res["b_saving_ms"] = round(res["b_reference_ms"] - res["b_ours_ms"], 2)
        rel = max(abs(float(a) - float(b)) / abs(float(b)) for a, b in zip(mel_o, mel_r))
        res["b_mel_loss_rel_diff"] = rel
        res["b_mel_loss_within_bar"] = rel <= 1e-6
    print(json.dumps(res))


if __name__ == "__main__":
    main()
