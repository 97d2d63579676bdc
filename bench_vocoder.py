"""Vocoder benchmark: this library's FireflyGAN (the reference's default vocoder) and Vocos, and the reference FireflyGAN
network in PyTorch on the same GPU, on one seeded mel batch (B = 32, n_mel = 128, T = 1000 frames by default).

    python bench_vocoder.py [--B 32] [--T 1000] [--steps 10] [--warmup-s 2]

Every arm: warm-up of at least --warmup-s seconds, then --steps timed calls, each after an L2 flush, timed with CUDA events
(every step is listed).  Reported per arm: ms per call, mel frames/s, audio-seconds/s at 44.1 kHz (512 samples per frame),
and for FireflyGAN the algorithmic and tensor-core-issued TFLOP/s, per-stage ms (st_profile_* classes) and the parity of
two utterances against the PyTorch arm.  The PyTorch arm runs the reference's own FireflyGANBase where
oracle/stage_ffgan.py has staged it under oracle/_ref (kind "reference"), else oracle/ffgan_ref.py (a restatement pinned
to the reference by tests/test_ffgan.py, kind "port"); its TF32 settings are recorded.  Writes nothing;
prints one JSON line."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

SR, HOP = 44100, 512


def head_gemms():
    """(name, stage, rows per mel frame, N, K, taps, algorithmic FLOPs per frame) of every conv-GEMM of the FireflyGAN."""
    from oracle import ffgan_ref as R
    out = [("stem", "backbone", 1, 128, 128, 7, 2 * 128 * 128 * 7)]
    for i, (d, depth) in enumerate(zip(R.DIMS, R.DEPTHS)):
        if i:
            out.append((f"down{i}", "backbone", 1, d, R.DIMS[i - 1], 1, 2 * d * R.DIMS[i - 1]))
        out += [(f"pw{i}", "backbone", 1, 4 * d, d, 1, 2 * 4 * d * d)] * depth + [(f"pw{i}b", "backbone", 1, d, 4 * d, 1, 2 * 4 * d * d)] * depth
    out.append(("conv_pre", "conv_pre", 1, 512, 512, 13, 2 * 512 * 512 * 13))
    spf = 1
    for i, (u, k) in enumerate(R.UPS):
        cin, c = 512 >> i, 512 >> (i + 1)
        out.append((f"ups{i}", f"stage{i}", spf, u * c, cin, 3, 2 * spf * u * c * cin * 2))   # 2 of the 3 packed taps are live
        spf *= u
        for kk in R.RES_K:
            out += [(f"res{i}", f"stage{i}", spf, c, c, kk, 2 * spf * c * c * kk)] * 6
    return out


def flops_per_frame():
    """algorithmic and issued (3 split-bf16 passes over the GEMM's N tile — 16 / 32 / 64 channels for outputs of exactly that
    width, else multiples of 128 — and 64-channel K blocks) FLOPs per mel frame, per stage; the dwconv / LayerNorm / post rows
    are counted as algorithmic only."""
    alg, issued = {}, {}
    for _, st, rows, N, K, taps, f in head_gemms():
        alg[st] = alg.get(st, 0) + f
        n_tile = N if N in (16, 32, 64) else math.ceil(N / 128) * 128
        issued[st] = issued.get(st, 0) + 3 * 2 * rows * n_tile * (math.ceil(K / 64) * 64) * taps
    alg["post"] = 2 * 512 * 16 * 13
    return alg, issued


class Timer:
    def __init__(self, dev):
        self.flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)      # > the 50 MB L2

    def run(self, fn, steps, warmup_s):
        t0 = time.perf_counter()
        n = 0
        while time.perf_counter() - t0 < warmup_s or n < 2:
            fn(); n += 1
            torch.cuda.synchronize()
        ms = []
        for _ in range(steps):
            self.flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return dict(warmup_calls=n, steps_ms=[round(x, 3) for x in ms], ms=float(sorted(ms)[len(ms) // 2]))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--T", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup-s", type=float, default=2.0)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vocoder.py measures on a CUDA device; none is available")
    import __graft_entry__ as ge
    ge.build()
    from oracle import ffgan_ref as R, vocoder_ref as V
    from stabletts_b200 import FireflyGANBase, Vocos, _lib
    dev = torch.device("cuda:0")
    B, T = args.B, args.T
    frames, audio_s = B * T, B * T * HOP / SR
    mel = R.make_mel(args.seed, B, T).to(dev)
    st = R.make_state()
    tm = Timer(dev)
    props = torch.cuda.get_device_properties(dev)
    res = dict(metric="vocoder", B=B, T=T, n_mel=128, gpu=props.name, torch=torch.__version__)
    try:
        import subprocess
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # noqa: BLE001
        res["power_limit"] = f"unknown ({e})"

    def rates(ms):
        return dict(ms=round(ms, 3), frames_per_s=round(frames / ms * 1e3, 1), audio_s_per_s=round(audio_s / ms * 1e3, 1))

    # ---- this library's FireflyGAN ----
    ff = FireflyGANBase().eval()
    ff.load_state_dict(st, strict=True)
    ff = ff.to(dev)
    out = {}
    r = tm.run(lambda: out.__setitem__("a", ff(mel)), args.steps, args.warmup_s)
    alg, issued = flops_per_frame()
    a_tot, i_tot = sum(alg.values()) * frames, sum(issued.values()) * frames
    arm = dict(kind="cuda", **rates(r["ms"]), steps_ms=r["steps_ms"], warmup_calls=r["warmup_calls"],
               alg_tflops=round(a_tot / r["ms"] / 1e9, 2), issued_tflops=round(i_tot / r["ms"] / 1e9, 2),
               gflop_per_frame=round(a_tot / frames / 1e9, 4), issued_over_alg=round(i_tot / a_tot, 3),
               workspace_gb=round(ff.workspace_bytes(B, T) / 1e9, 2))
    lib, h = _lib.load_library(), ff._handle
    lib.st_profile_begin(h)
    ff(mel)
    n = _lib.ST_PROF_NCAT
    ms_a, fl_a, by_a, ln_a = (C.c_double * n)(), (C.c_double * n)(), (C.c_double * n)(), (C.c_int64 * n)()
    _lib.check(lib, h, lib.st_profile_end(h, ms_a, fl_a, by_a, ln_a), "st_profile_end")
    stages = {}
    for i, name in enumerate(_lib.ST_PROF_NAMES):
        if name.startswith("ffgan_"):
            key = name[len("ffgan_"):]
            ms_i = ms_a[i]
            a_i = alg.get(key, 0) * frames
            stages[key] = dict(ms=round(ms_i, 3), launches=int(ln_a[i]), alg_tflops=round(a_i / ms_i / 1e9, 2) if ms_i else None,
                               issued_tflops=round(issued.get(key, 0) * frames / ms_i / 1e9, 2) if ms_i else None)
    arm["stages"] = stages
    arm["stages_note"] = ("per-launch CUDA events in a separate call (profiled, so the sum exceeds ms); stageN = ups[N] + "
                          "ParralelBlock N; issued = 3 split-bf16 passes x the N tile (16 / 32 / 64 or 128-multiples) x 64-channel K blocks")
    res["ffgan"] = arm
    audio = out["a"]

    # ---- the PyTorch arm on the same GPU: the reference's own module when oracle/stage_ffgan.py staged it, else the
    #      oracle restatement ----
    from oracle import stage_ffgan
    sd = {k: v.to(dev) for k, v in st.items()}
    if stage_ffgan.available():
        ref_model = stage_ffgan.load_reference()().eval()
        ref_model.load_state_dict(sd, strict=True)
        ref_model = ref_model.to(dev)
        kind, ref_fn = "reference", lambda x: ref_model(x)
    else:
        kind, ref_fn = "port", lambda x: R.ffgan_forward(sd, x)
    tf32, mm_tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    with torch.inference_mode():
        r = tm.run(lambda: ref_fn(mel), max(2, args.steps // 2), args.warmup_s)
        res["pytorch"] = dict(kind=kind, cudnn_allow_tf32=tf32, matmul_allow_tf32=mm_tf32,
                              **rates(r["ms"]), steps_ms=r["steps_ms"], warmup_calls=r["warmup_calls"])
        # parity reference: the same network in fp32 without TF32, two utterances
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        rows = [0, B - 1]
        ref = ref_fn(mel[rows])
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32, mm_tf32
    d = (audio[rows].double() - ref.double())
    res["ffgan"]["parity"] = dict(max_rel=float(d.abs().max() / ref.abs().max()), l2_rel=float(d.norm() / ref.double().norm()),
                                  rows=rows, vs=f"the PyTorch arm ({kind}) in fp32 on the GPU, TF32 off")
    del sd, ref, out, audio
    ff.release()
    torch.cuda.empty_cache()

    # ---- this library's Vocos on the same mel ----
    voc = Vocos(**V.DIMS).eval()
    voc.load_state_dict(V.make_state(), strict=True)
    voc = voc.to(dev)
    r = tm.run(lambda: voc(mel), args.steps, args.warmup_s)
    res["vocos"] = dict(kind="cuda", **rates(r["ms"]), steps_ms=r["steps_ms"], warmup_calls=r["warmup_calls"])
    res["ffgan_speedup_vs_pytorch"] = round(res["pytorch"]["ms"] / res["ffgan"]["ms"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
