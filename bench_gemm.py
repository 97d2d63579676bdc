"""Per-shape benchmark of the 256-channel wgmma conv-GEMM at the flagship workload's shapes (bench.py cfg1: 32 utterances
doubled to BB = 64 rows by classifier-free guidance, T = 1000 frames, hidden 256, filter 1024).  Prints one JSON line per
shape, then one line with the GPU it ran on.

    python bench_gemm.py [--reps R] [--repeats N]

Shapes (st_bench_conv on device-generated operands; the epilogue of the call site, or the closest one the hook offers):
  qkv        256 -> 768, 1 tap, bias, split-bf16 planes out (the product adds the RoPE; same tile loop)
  o          256 -> 256, 1 tap, residual + fused LayerNorm / modulate
  conv_1     256 -> 1024, 3 taps, bias + SiLU + mask
  conv_2     1024 -> 256, 3 taps, residual + fused LayerNorm / modulate
  long_skip  512 -> 256, 3 taps, bias (the product reads two 256-channel sources; same K loop)
QKV and O run in split-bf16 ("bf16x3", three MMAs per k-step); the FFN and long-skip convs run in both precisions, as the
two modes of bench.py do ("fp16x2", two MMAs per k-step, is the default).

Per shape: `ms` is the median over --repeats timings, each the mean of --reps back-to-back launches between CUDA events after
a warm-up.  `tflops_alg` counts 2 * BB * T * N * K * taps; `tflops_issued` counts what the tensor cores execute: every
128-frame tile of the launch (padded frames included) times the MMAs per k-step.  `l2_to_sm_bytes` follows the tile
schedule the library reports (st_test_gemm_ex's plan): per tile and 64-wide k-block one A box (16 KB per operand plane)
plus both weight planes' BN x 64 tile.  `hbm_bytes` is the compulsory traffic from the shapes: operand planes and weights
read once, outputs written once, residual rows read once.  The card's name, power limit and SM clocks are read in the same run.  Nothing is written to the
tree."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

BB, T, H, FILTER = 64, 1000, 256, 1024
BLOCK_M, BLOCK_K = 128, 64
# name, Cin, Cout, taps, st_bench_conv epilogue (0 bias, 2 SiLU, 3 residual + LayerNorm), precisions
SHAPES = [("qkv", H, 3 * H, 1, 0, (0,)), ("o", H, H, 1, 3, (0,)), ("conv_1", H, FILTER, 3, 2, (1, 0)),
          ("conv_2", FILTER, H, 3, 3, (1, 0)), ("long_skip", 2 * H, H, 3, 0, (1, 0))]
PREC_NAMES = ("bf16x3", "fp16x2")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit": q[1], "max_sm_clock": q[2], "sm_clock_after_timing": q[3]}
    except Exception as e:                                       # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({e})", "max_sm_clock": "unavailable",
                "sm_clock_after_timing": "unavailable"}


def plan_of(lib, h, cin, cout, taps, epi, prec, dev):
    """the launch the library makes for this shape (tile width, grid), from one st_test_gemm_ex call"""
    from stabletts_b200 import _lib
    z = lambda *s: torch.zeros(*s, device=dev)                  # noqa: E731
    t = {"A0": z(BB, T, cin), "W": z(taps, cout, cin), "bias": z(cout), "mask": torch.ones(BB, T, device=dev),
         "gate": z(BB, cout), "resid": z(BB, T, cout), "ln_shift": z(BB, cout), "ln_scale": z(BB, cout)}
    plane = lambda: torch.zeros(BB, T, cout, device=dev, dtype=torch.float16 if prec else torch.bfloat16)   # noqa: E731
    hi, lo = ("u_hi", "u_lo") if epi == 3 else ("out_hi", "out_lo")    # the LayerNorm output, or the output planes
    o = {"out_f32": z(BB, T, cout), hi: plane()}
    if not prec:
        o[lo] = plane()
    d = _lib.StTestGemmDesc()
    for k, v in {**t, **o}.items():
        setattr(d, k, v.data_ptr())
    flags = {0: 1, 2: 1 | 2 | 8, 3: 8 | 16 | 32}[epi]
    for k, v in dict(B=BB, BB=BB, T=T, a_bmod=BB, n_src=1, C0=cin, C1=0, N=cout, taps=taps, dil=1, flags=flags,
                     c_clamp=BB - 1, resid_clamp=BB - 1, film_H=cout, gate_bstride=cout, ada_bstride=cout, ln=int(epi == 3),
                     prec=prec, out16=prec if epi != 3 else 0, u16=prec if epi == 3 else 0, ksplit=1, num_sms=0).items():
        setattr(d, k, v)
    plan = _lib.StTestGemmPlan()
    _lib.check(lib, h, lib.st_test_gemm_ex(h, C.byref(d), C.byref(plan), torch.cuda.current_stream().cuda_stream),
               "st_test_gemm_ex")
    torch.cuda.synchronize()
    return plan


def traffic(cin, cout, taps, epi, prec, bn):
    tiles = BB * -(-T // BLOCK_M) * (cout // bn)
    num_kb = taps * -(-cin // BLOCK_K)
    a_box = (1 if prec else 2) * BLOCK_M * BLOCK_K * 2
    w_tile = 2 * bn * BLOCK_K * 2                                # hi + lo planes
    l2 = tiles * num_kb * (a_box + w_tile)
    plane = 2 if prec else 4                                     # bytes per element: one fp16 plane, or bf16 hi + lo
    out = {0: plane, 2: plane, 3: 4 + 4 + plane}[epi]            # planes; or residual read + fp32 out + LayerNorm planes
    hbm = BB * T * cin * plane + taps * cout * cin * 4 + BB * T * cout * out
    issued = 2.0 * tiles * BLOCK_M * bn * cin * taps * (2 if prec else 3)
    return l2, hbm, issued


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50, help="launches per timing (>= 50)")
    ap.add_argument("--repeats", type=int, default=5, help="timings per shape; the median is reported")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm.py measures on a CUDA device; none is present")
    from stabletts_b200 import _lib
    dev = torch.device("cuda:0")
    lib = _lib.load_library()
    h = C.c_void_p()
    _lib.check(lib, None, lib.st_create_ffgan(0, C.byref(h)), "st_create_ffgan")
    _lib.check(lib, h, lib.st_set_engine(h, _lib.ST_ENGINE_TCGEN05), "st_set_engine")
    try:
        for name, cin, cout, taps, epi, precs in SHAPES:
            for prec in precs:
                plan = plan_of(lib, h, cin, cout, taps, epi, prec, dev)
                ms = C.c_float()
                _lib.check(lib, h, lib.st_bench_conv(h, BB, cin, cout, T, taps, epi, prec, 10, C.byref(ms)), "st_bench_conv")
                runs = []
                for _ in range(args.repeats):
                    _lib.check(lib, h, lib.st_bench_conv(h, BB, cin, cout, T, taps, epi, prec, max(50, args.reps), C.byref(ms)),
                               "st_bench_conv")
                    runs.append(ms.value)
                t = sorted(runs)[len(runs) // 2]
                l2, hbm, issued = traffic(cin, cout, taps, epi, prec, plan.bn)
                alg = 2.0 * BB * T * cout * cin * taps
                print(json.dumps({"shape": name, "precision": PREC_NAMES[prec], "BB": BB, "T": T, "Cin": cin, "Cout": cout,
                                  "taps": taps, "bn": plan.bn, "grid": plan.grid, "ms": round(t, 4),
                                  "ms_runs": [round(x, 4) for x in runs], "tflops_alg": round(alg / t / 1e9, 1),
                                  "tflops_issued": round(issued / t / 1e9, 1), "l2_to_sm_bytes": l2,
                                  "l2_to_sm_tb_per_s": round(l2 / t / 1e9, 2), "hbm_bytes": hbm,
                                  "hbm_tb_per_s": round(hbm / t / 1e9, 3)}), flush=True)
    finally:
        lib.st_destroy(h)
    print(json.dumps(gpu_info()), flush=True)


if __name__ == "__main__":
    main()
