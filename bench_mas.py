"""Monotonic alignment search and the training forward's losses on the GPU against the reference.  Prints one JSON line.

    python bench_mas.py [--iters 20] [--warmup 3] [--steps 6]

- ``maximum_path``: stabletts_b200's at B = 32, T_y = 1000, T_x = 400 (the trainer's batch in DistributedBucketSampler's
  largest bucket) with a full mask and with ragged lengths drawn from the buckets, timed with CUDA events after a warm-up;
  the reference's (numba, from the staged oracle/_ref copy) on the same CUDA tensors, timed on the host clock — it copies
  to the host and back and so synchronises itself.  "not measured" when numba or the staged copy is missing.
- ``compute_losses`` against the reference ``StableTTS.forward`` in eval mode under no_grad on the same GPU.
- The reference's own training step (forward + backward, train mode) at B = 32 in its largest bucket with numba's
  ``maximum_path`` and with the drop-in, alternated, from the same seed: the losses must be bitwise equal.
The card's name and power limit are read in the same run.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

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


def host_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / iters


def scores_batch(gen, B, Ty, Tx, dev, D=80):
    mu = torch.randn(B, D, Tx, generator=gen)
    tok = torch.sort(torch.randint(0, Tx, (B, Ty), generator=gen), dim=1).values
    y = torch.gather(mu, 2, tok[:, None, :].expand(B, D, Ty)) + torch.randn(B, D, Ty, generator=gen)
    nc = -0.5 * (y * y).sum(1)[:, :, None] + torch.einsum("bdt,bds->bts", y, mu) - 0.5 * (mu * mu).sum(1)[:, None, :]
    return nc.to(dev)


def prefix_mask(t_y, t_x, Ty, Tx, dev):
    return ((torch.arange(Ty)[None, :, None] < t_y[:, None, None]) & (torch.arange(Tx)[None, None, :] < t_x[:, None, None])).float().to(dev)


def load_reference_mas():
    from oracle import stage_mas
    try:
        return stage_mas.load_reference(), None
    except Exception as e:                                   # noqa: BLE001 — numba or the staged copy missing
        return None, f"not measured ({type(e).__name__}: {e})"


def training_inputs(gen, B, Tx, Ty, Tz, n_mel, dev):
    from oracle import synth_ref
    ids, x_lengths, z = synth_ref.make_inputs(int(torch.randint(0, 10 ** 6, (1,), generator=gen)), [Tx] * B, Tz, n_mel)
    x_lengths = torch.randint(Tx // 2, Tx + 1, (B,), generator=gen)
    x_lengths[0] = Tx
    ids = ids * (torch.arange(Tx)[None] < x_lengths[:, None])
    y_lengths = torch.maximum(torch.randint(Ty * 3 // 4, Ty + 1, (B,), generator=gen), x_lengths)
    y_lengths[0] = Ty
    y = (torch.randn(B, n_mel, Ty, generator=gen) * 2.0 - 4.0) * (torch.arange(Ty)[None] < y_lengths[:, None])[:, None]
    z_lengths = torch.full((B,), Tz)
    return [t.to(dev) for t in (ids, x_lengths, y, y_lengths, z, z_lengths)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=6, help="training steps per arm (alternated)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mas.py needs a CUDA device")
    from stabletts_b200 import StableTTS, monotonic_align
    dev = torch.device("cuda:0")
    name, limit = card()
    res = {"metric": "mas", "gpu": name, "power_limit": limit}
    gen = torch.Generator().manual_seed(0)
    B, Ty, Tx = 32, 1000, 400

    # ---- maximum_path ----------------------------------------------------------------------------------------------
    nc = scores_batch(gen, B, Ty, Tx, dev)
    full = torch.ones(B, Ty, Tx, device=dev)
    t_y = torch.randint(600, Ty + 1, (B,), generator=gen)
    t_x = torch.minimum(torch.randint(150, Tx + 1, (B,), generator=gen), t_y)
    ragged = prefix_mask(t_y, t_x, Ty, Tx, dev)
    res["maximum_path_ms"] = {"b32_1000x400_full": cuda_ms(lambda: monotonic_align.maximum_path(nc, full), args.iters, args.warmup),
                              "b32_1000x400_ragged": cuda_ms(lambda: monotonic_align.maximum_path(nc, ragged), args.iters, args.warmup)}
    ref_mas, why = load_reference_mas()
    if ref_mas is None:
        res["reference_maximum_path_ms"] = why
    else:
        n = max(3, args.iters // 4)
        res["reference_maximum_path_ms"] = {
            "b32_1000x400_full": host_ms(lambda: ref_mas.maximum_path(nc, full), n, 1),
            "b32_1000x400_ragged": host_ms(lambda: ref_mas.maximum_path(nc, ragged), n, 1)}
        res["maximum_path_bitwise_equal"] = bool(torch.equal(ref_mas.maximum_path(nc, full), monotonic_align.maximum_path(nc, full))
                                                 and torch.equal(ref_mas.maximum_path(nc, ragged),
                                                                 monotonic_align.maximum_path(nc, ragged)))

    # ---- compute_losses and the reference training step ----------------------------------------------------------------
    from oracle import stage_synth, synth_ref
    if ref_mas is None or not stage_synth.available():
        res["compute_losses_ms"] = res["reference_forward_eval_ms"] = res["training_step_ms"] = "not measured (reference not staged)"
        print(json.dumps(res))
        return
    RefStableTTS = stage_synth.load_reference()
    import models.model as ref_model
    n_mel = 80
    st = synth_ref.make_state(n_mel=n_mel)
    ours = StableTTS(synth_ref.N_VOCAB, n_mel, 256, 1024, 4, 3, 6, 3, 0.1, 256).eval()
    ours.load_state_dict(st, strict=True)
    ours = ours.to(dev)
    ref = RefStableTTS(synth_ref.N_VOCAB, n_mel, 256, 1024, 4, 3, 6, 3, 0.1, 256)
    ref.load_state_dict(st, strict=True)
    ref = ref.to(dev)
    inp = training_inputs(gen, B, 300, Ty, 200, n_mel, dev)
    ref_model.monotonic_align = ref_mas
    ref.eval()
    with torch.no_grad():
        res["reference_forward_eval_ms"] = host_ms(lambda: ref(*inp), max(3, args.iters // 4), 1)
    res["compute_losses_ms"] = host_ms(lambda: ours.compute_losses(*inp), args.iters, args.warmup)

    ref.train()
    opt_params = [p for p in ref.parameters() if p.requires_grad]

    def step(mas):
        ref_model.monotonic_align = mas
        torch.manual_seed(1234)
        for p in opt_params:
            p.grad = None
        dur, diff, prior, _ = ref(*inp)
        (dur + diff + prior).backward()
        return torch.stack([dur.detach(), diff.detach(), prior.detach()])

    arms = {"numba": ref_mas, "stabletts_b200": monotonic_align}
    times = {k: [] for k in arms}
    losses, repeat_equal = {}, True
    for k in arms:                                           # warm-up (numba JIT, cuBLAS / cuDNN algorithm choice)
        losses[k] = step(arms[k])
    torch.cuda.synchronize()
    for _ in range(args.steps):
        for k, mas in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = step(mas)
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
            repeat_equal = repeat_equal and bool(torch.equal(out, losses[k]))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    res["training_step_ms"] = {"shape": f"B={B} T_y={Ty} T_x=300 train mode, forward + backward", **med,
                               "speedup": med["numba"] / med["stabletts_b200"]}
    res["training_losses_bitwise_equal"] = bool(torch.equal(losses["numba"], losses["stabletts_b200"]))
    res["training_losses"] = losses["numba"].tolist()
    res["training_losses_repeatable"] = repeat_equal
    print(json.dumps(res))


if __name__ == "__main__":
    main()
