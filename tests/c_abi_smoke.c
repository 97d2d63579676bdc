/* Pure-C consumer of the C ABI (include/stabletts_b200.h): no Python, no torch types anywhere.
 *   gcc tests/c_abi_smoke.c -Iinclude -I/usr/local/cuda/include -Lstabletts_b200 -lstabletts_b200 \
 *       -L/usr/local/cuda/lib64 -lcudart -lm -o build/c_abi_smoke
 * Without a GPU it checks that st_create fails loudly (no CPU fallback) and exits 0.
 * On an H100 it loads seeded synthetic weights under the reference's 116 parameter names, runs a 4-step Euler
 * CFG solve on a padded batch and checks: finite output, exact zeros at masked frames, determinism. */
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "stabletts_b200.h"

static uint32_t g_seed = 12345u;
static float frand(void) { g_seed = g_seed * 1664525u + 1013904223u; return ((g_seed >> 8) & 0xFFFFFF) / 8388608.0f - 1.0f; }

static float* dev_random(size_t n, float scale) {
    float* h = (float*)malloc(n * sizeof(float));
    for (size_t i = 0; i < n; ++i) h[i] = frand() * scale;
    float* d = NULL;
    if (cudaMalloc((void**)&d, n * sizeof(float)) != cudaSuccess) { fprintf(stderr, "cudaMalloc failed\n"); exit(2); }
    cudaMemcpy(d, h, n * sizeof(float), cudaMemcpyHostToDevice);
    free(h);
    return d;
}

static int load(st_handle* h, const char* name, size_t n, size_t fan_in) {
    float* d = dev_random(n, 1.0f / sqrtf((float)fan_in));
    int rc = st_load_weight(h, name, d, (int64_t)n, NULL);
    cudaDeviceSynchronize();
    cudaFree(d);
    if (rc) fprintf(stderr, "st_load_weight(%s): %s\n", name, st_last_error(h));
    return rc;
}

static int load_wb(st_handle* h, const char* base, size_t out, size_t in, size_t k) {
    char nm[160];
    snprintf(nm, sizeof nm, "%s.weight", base);
    if (load(h, nm, out * in * k, in * k)) return 1;
    snprintf(nm, sizeof nm, "%s.bias", base);
    return load(h, nm, out, in * k);
}

int main(void) {
    const int M = 80, H = 256, F = 1024, L = 6, K = 3;
    st_dims dims = {M, H, F, 4, L, K, H};
    st_handle* h = NULL;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        int rc = st_create(&dims, 0, &h);
        printf("no CUDA device: st_create rc=%d (\"%s\")\n", rc, st_last_error(NULL));
        return rc != 0 ? 0 : 1;                       /* must fail loudly: no CPU fallback */
    }
    if (st_create(&dims, 0, &h)) { fprintf(stderr, "st_create: %s\n", st_last_error(NULL)); return 1; }
    printf("library version %d\n", st_version());
    char nm[160];
    int bad = 0;
    bad |= load_wb(h, "time_mlp.layer.0", F, H, 1);
    bad |= load_wb(h, "time_mlp.layer.2", H, F, 1);
    bad |= load_wb(h, "in_proj", H, H + M, 1);
    for (int i = 0; i < L; ++i) {
        const char* conv[4] = {"q", "k", "v", "o"};
        snprintf(nm, sizeof nm, "blocks.%d.time_fusion.film", i); bad |= load_wb(h, nm, 2 * H, H, 1);
        for (int c = 0; c < 4; ++c) { snprintf(nm, sizeof nm, "blocks.%d.block.attn.conv_%s", i, conv[c]); bad |= load_wb(h, nm, H, H, 1); }
        snprintf(nm, sizeof nm, "blocks.%d.block.mlp.conv_1", i); bad |= load_wb(h, nm, F, H, K);
        snprintf(nm, sizeof nm, "blocks.%d.block.mlp.conv_2", i); bad |= load_wb(h, nm, H, F, K);
        snprintf(nm, sizeof nm, "blocks.%d.block.adaLN_modulation.2", i); bad |= load_wb(h, nm, 6 * H, H, 1);
    }
    bad |= load_wb(h, "final_proj", M, H, 1);
    bad |= load_wb(h, "cond_proj.0", F, M, K);
    bad |= load_wb(h, "cond_proj.2", F, F, K);
    bad |= load_wb(h, "cond_proj.4", H, F, K);
    for (int i = 0; i < L / 2; ++i) { snprintf(nm, sizeof nm, "lsc_layers.%d", i); bad |= load_wb(h, nm, H, 2 * H, K); }
    if (bad) return 1;
    if (st_finalize_weights(h, NULL)) { fprintf(stderr, "finalize: %s\n", st_last_error(h)); return 1; }

    const int B = 2, T = 50, len[2] = {50, 31}, steps = 4;
    float* mu = dev_random((size_t)B * M * T, 1.f);
    float* c = dev_random((size_t)B * H, 1.f);
    float* fc = dev_random(M, 1.f);
    float* fs = dev_random(H, 1.f);
    float* z0 = dev_random((size_t)B * M * T, 1.f);
    float hm[2 * 50];
    for (int b = 0; b < B; ++b) for (int t = 0; t < T; ++t) hm[b * T + t] = t < len[b] ? 1.f : 0.f;
    float* mask; cudaMalloc((void**)&mask, sizeof hm); cudaMemcpy(mask, hm, sizeof hm, cudaMemcpyHostToDevice);
    float tspan[5]; for (int i = 0; i <= steps; ++i) tspan[i] = (float)i / steps;
    const size_t n = (size_t)B * M * T;
    float *z, *out1 = (float*)malloc(n * 4), *out2 = (float*)malloc(n * 4);
    cudaMalloc((void**)&z, n * 4);
    for (int rep = 0; rep < 2; ++rep) {
        cudaMemcpy(z, z0, n * 4, cudaMemcpyDeviceToDevice);
        if (st_solve(h, z, mu, mask, c, fc, fs, 3.0f, tspan, steps, ST_EULER, B, T, NULL)) { fprintf(stderr, "st_solve: %s\n", st_last_error(h)); return 1; }
        if (cudaDeviceSynchronize() != cudaSuccess) { fprintf(stderr, "device error: %s\n", cudaGetErrorString(cudaGetLastError())); return 1; }
        cudaMemcpy(rep ? out2 : out1, z, n * 4, cudaMemcpyDeviceToHost);
    }
    int ok = 1; double s = 0;
    for (size_t i = 0; i < n; ++i) { if (!isfinite(out1[i])) ok = 0; s += fabs(out1[i]); }
    if (memcmp(out1, out2, n * 4) != 0) { printf("NOT deterministic\n"); ok = 0; }
    /* the sample is z + sum dt*v with v == 0 at masked frames: masked frames keep their initial noise */
    float* hz0 = (float*)malloc(n * 4); cudaMemcpy(hz0, z0, n * 4, cudaMemcpyDeviceToHost);
    for (int m = 0; m < M; ++m) for (int t = len[1]; t < T; ++t) if (out1[((size_t)1 * M + m) * T + t] != hz0[((size_t)1 * M + m) * T + t]) ok = 0;
    printf("solve: mean|x| = %.4f, launches = %lld, %s\n", s / n, (long long)st_launch_count(h), ok ? "OK" : "FAILED");
    st_destroy(h);
    return ok ? 0 : 1;
}
