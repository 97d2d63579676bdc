"""Benchmark of StableTTS.synthesise (text + reference mel -> mel) on this library's kernels, per stage, against the
reference's own StableTTS.synthesise in PyTorch on the same GPU.  Prints one JSON line.

    python bench_synthesise.py [--steps K] [--warmup W]

Workloads (seeded weights and inputs, 128 mel channels, 10-step Euler, CFG 3.0):
  api  B = 1: one utterance of 129 interspersed tokens and a 430-frame (5 s) reference mel — the call api.py makes
  b32  B = 32: ragged text of 60-200 tokens
Per stage, CUDA events around each module call (median over K): style encoder, text encoder, duration predictor,
alignment (including its host read of the output length) and the CFM solve; the total is a host clock around the whole
synthesise call ending in a device synchronise.  The reference arm is the staged reference StableTTS (oracle/_ref, made by
build() where a checkout exists; `kind: "reference"`) or else the oracle restatement (`kind: "port"`), with TF32 off and
the same initial noise z; `parity` is the max-rel difference of the two arms' mels.  The GPU's name, power limit and
maximum SM clock are read in the same run.  Nothing is written to the tree."""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

N_MEL, T_REF, STEPS, CFG = 128, 430, 10, 3.0


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit": q[1], "max_sm_clock": q[2]}
    except Exception as e:                                       # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({e})", "max_sm_clock": "unavailable"}


def workloads():
    g = torch.Generator().manual_seed(5)
    return {"api": [129], "b32": [int(v) for v in torch.randint(60, 201, (32,), generator=g)]}


@contextlib.contextmanager
def injected_noise(z):
    """the reference draws z = randn_like(mu_y) * temperature (models/flow_matching.py:45): hand it the same z"""
    orig = torch.randn_like
    torch.randn_like = lambda t, **kw: z.to(device=t.device, dtype=t.dtype).clone()
    try:
        yield
    finally:
        torch.randn_like = orig


def stage_times(model, ids, lens, y, z):
    """one synthesise, stage by stage (the calls StableTTS.synthesise makes), timed with CUDA events"""
    from stabletts_b200 import expand_by_durations
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    with torch.inference_mode():
        ev[0].record()
        c = model.ref_encoder(y, None)
        ev[1].record()
        x, mu_x, x_mask = model.encoder(ids, c, lens)
        ev[2].record()
        logw = model.dp(x, x_mask, c)
        ev[3].record()
        mu_y, y_mask, y_lengths, _ = expand_by_durations(logw, x_mask, mu_x, 1.0, return_attn=True)
        ev[4].record()
        cfg = {"fake_speaker": model.fake_speaker, "fake_content": model.fake_content, "cfg_strength": CFG}
        model.decoder(mu_y, y_mask, STEPS, 1.0, c, "euler", cfg, z=z)
        ev[5].record()
    torch.cuda.synchronize()
    names = ("style_encoder", "text_encoder", "duration_predictor", "alignment", "cfm_solve")
    return {n: ev[i].elapsed_time(ev[i + 1]) for i, n in enumerate(names)}


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_synthesise.py measures on a CUDA device; none is present")
    from oracle import stage_synth, synth_ref
    from stabletts_b200 import StableTTS
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    state = synth_ref.make_state(n_mel=N_MEL)
    ours = StableTTS(synth_ref.N_VOCAB, N_MEL, 256, 1024, 4, 3, 6, 3, 0.1, 256).eval()
    ours.load_state_dict(state, strict=True)
    ours = ours.to(dev)
    kind = "reference" if stage_synth.available() else "port"
    ref_model = None
    if kind == "reference":
        Ref = stage_synth.load_reference()
        ref_model = Ref(synth_ref.N_VOCAB, N_MEL, 256, 1024, 4, 3, 6, 3, 0.1, 256).eval()
        ref_model.load_state_dict(state, strict=True)
        ref_model = ref_model.to(dev)
    result = {"bench": "synthesise", "solver": f"euler x {STEPS}, cfg {CFG}", "n_mel": N_MEL, "reference_kind": kind, **gpu_info()}
    for wname, lens in workloads().items():
        # durations are discontinuous (ceil(exp(logw))): take the first input seed whose every token is 5e-4 w clear of an
        # integer, so that both arms agree on the alignment and the mels can be compared frame by frame (at B = 32 with
        # thousands of tokens no seed may clear it: the last seed is kept and `duration_margin` says so)
        for seed in range(17, 81):
            ids, lens_t, y = (v.to(dev) for v in synth_ref.make_inputs(seed, lens, T_REF, N_MEL))
            with torch.inference_mode():
                c = ours.ref_encoder(y, None)
                x, _, x_mask = ours.encoder(ids, c, lens_t)
                w = (torch.exp(ours.dp(x, x_mask, c)) * x_mask).double()
            margin = bool((((w - w.round()).abs() >= 5e-4 * w) | (x_mask == 0)).all())
            if margin:
                break
        with torch.inference_mode():
            probe = ours.synthesise(ids, lens_t, 1, 1.0, y, 1.0, "euler", CFG)
        Ty = probe["attn"].shape[-1]
        frames = int(probe["attn"].sum())
        z = torch.randn(len(lens), N_MEL, Ty, generator=torch.Generator().manual_seed(23)).to(dev)
        for _ in range(args.warmup):
            stage_times(ours, ids, lens_t, y, z)
            with torch.inference_mode():
                ours.synthesise(ids, lens_t, STEPS, 1.0, y, 1.0, "euler", CFG, z=z)
        stages = [stage_times(ours, ids, lens_t, y, z) for _ in range(max(1, args.steps))]
        walls = []
        for _ in range(max(1, args.steps)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.inference_mode():
                out = ours.synthesise(ids, lens_t, STEPS, 1.0, y, 1.0, "euler", CFG, z=z)
            torch.cuda.synchronize()
            walls.append((time.perf_counter() - t0) * 1e3)
        # reference arm: the same weights, inputs and z
        ref_walls = []
        for i in range(1 + max(1, min(args.steps, 3))):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.inference_mode(), injected_noise(z):
                if ref_model is not None:
                    ref = ref_model.synthesise(ids, lens_t, STEPS, 1.0, y, 1.0, "euler", CFG)
                else:
                    ref = synth_ref.synthesise(state, ids.cpu(), lens_t.cpu(), STEPS, y.cpu(), z.cpu(), 1.0, "euler", CFG)
            torch.cuda.synchronize()
            if i:                                                # the first call warms up
                ref_walls.append((time.perf_counter() - t0) * 1e3)
        same_len = tuple(ref["attn"].shape) == tuple(out["attn"].shape) and bool(torch.equal(ref["attn"].cpu().float(), out["attn"].cpu()))
        a, b = out["decoder_outputs"].double().cpu(), ref["decoder_outputs"].double().cpu()
        parity = float((a - b).abs().max() / b.abs().max()) if same_len else None
        total = median(walls)
        result[wname] = {
            "B": len(lens), "input_seed": seed, "duration_margin": margin, "tokens": sum(lens), "mel_frames": frames, "T_y": Ty,
            "stage_ms": {k: round(median([s[k] for s in stages]), 3) for k in stages[0]},
            "synthesise_ms": round(total, 3), "mel_frames_per_s": round(frames / (total / 1e3), 1),
            "reference_ms": round(median(ref_walls), 3), "speedup": round(median(ref_walls) / total, 3),
            "parity_max_rel": parity, "same_alignment": same_len,
        }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
