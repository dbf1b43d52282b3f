// trace_harness.cu - timeline of a chain of back-to-back GEMVs (C ABI, PDL, CUDA graph).  Links a -DSQLLM_TRACE build of
// the library (squeezellm_b200/csrc/*.cu).  Prints, per launch, min/max over CTAs of each phase stamp relative to the chain start (ns).
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -DSQLLM_TRACE -I include -o trace_harness \
//        tests/perf/trace_harness.cu squeezellm_b200/csrc/*.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include <algorithm>
#include "sqllm_b200.h"
extern "C" void sqllm_debug_set_trace(unsigned long long *buf, size_t stride_words);
extern "C" int sqllm_debug_last_grid(void);
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

int main(int argc, char **argv) {
    setvbuf(stdout, NULL, _IONBF, 0);
    const int bits = argc > 1 ? atoi(argv[1]) : 4, K = argc > 2 ? atoi(argv[2]) : 4096, N = argc > 3 ? atoi(argv[3]) : 4096;
    const int chain = argc > 4 ? atoi(argv[4]) : 12, use_graph = argc > 5 ? atoi(argv[5]) : 1;
    const int sparse = argc > 6 ? atoi(argv[6]) : 0;  // 1: CSR (0.45 %) + 10 zero dense rows, accumulate; 2: same, fused fp16

    const size_t qwords = (size_t)K / 32 * bits * N;
    // enough distinct copies that the chain never finds a matrix in L2 (>= 400 MB in rotation, 8x the 50 MB L2 of an H100)
    const int copies = (int)std::min<size_t>(40, std::max<size_t>(3, (400u << 20) / (qwords * 4) + 1));
    uint32_t *q; float *lut, *x, *y; unsigned long long *trace;
    CK(cudaMalloc(&q, qwords * 4 * copies)); CK(cudaMemset(q, 0x5a, qwords * 4 * copies));
    // every launch of the chain gets its own weights AND its own look-up table / outlier arrays: a decode step never finds a layer's small
    // arrays in L2 either (one shared table made the chain faster per launch than the real step)
    const size_t lutn = (size_t)N * 16;
    CK(cudaMalloc(&lut, lutn * 4 * copies)); CK(cudaMemset(lut, 0, lutn * 4 * copies));
    CK(cudaMalloc(&x, K * 4)); CK(cudaMemset(x, 0, K * 4));
    CK(cudaMalloc(&y, (size_t)N * 4 * chain)); CK(cudaMemset(y, 0, (size_t)N * 4 * chain));
    const size_t stride = 1024 * 32;
    CK(cudaMalloc(&trace, stride * 8 * chain)); CK(cudaMemset(trace, 0, stride * 8 * chain));
    size_t rstride = 0, nstride = 0, fstride = 0;
    int *rows = nullptr, *cols = nullptr, *fri = nullptr; float *vals = nullptr, *fr = nullptr; void *ws = nullptr; size_t wsb = 0; void *xh = nullptr, *yh = nullptr;
    if (sparse) {
        const int per = (int)(0.0045 * K + 0.5); const size_t nnz = (size_t)per * N;
        std::vector<int> hr(N + 1), hc(nnz);
        for (int c = 0; c <= N; ++c) hr[c] = c * per;
        for (size_t i = 0; i < nnz; ++i) hc[i] = (int)((i * 2654435761u) % K);
        rstride = ((size_t)N + 1 + 63) / 64 * 64; nstride = (nnz + 63) / 64 * 64; fstride = (size_t)K * 10;
        CK(cudaMalloc(&rows, rstride * 4 * copies)); CK(cudaMalloc(&cols, nstride * 4 * copies)); CK(cudaMalloc(&vals, nstride * 4 * copies));
        CK(cudaMemset(vals, 0, nstride * 4 * copies));
        for (int c = 0; c < copies; ++c) {
            CK(cudaMemcpy(rows + c * rstride, hr.data(), (N + 1) * 4, cudaMemcpyHostToDevice));
            CK(cudaMemcpy(cols + c * nstride, hc.data(), nnz * 4, cudaMemcpyHostToDevice));
        }
        CK(cudaMalloc(&fr, fstride * 4 * copies)); CK(cudaMemset(fr, 0, fstride * 4 * copies));
        CK(cudaMalloc(&fri, 40)); CK(cudaMemset(fri, 0, 40));
        wsb = 16u << 20; CK(cudaMalloc(&ws, wsb)); CK(cudaMemset(ws, 0, wsb));
        CK(cudaMalloc(&xh, K * 2)); CK(cudaMemset(xh, 0, K * 2)); CK(cudaMalloc(&yh, (size_t)N * 2 * chain));
    }
    cudaStream_t st; CK(cudaStreamCreate(&st));
    auto run_chain = [&](bool tr) {
        sqllm_debug_set_trace(tr ? trace : nullptr, tr ? stride : 0);
        for (int i = 0; i < chain; ++i) {
            sqllm_lutgemv_args a; memset(&a, 0, sizeof(a));
            a.bits = bits; a.in_features = K; a.out_features = N; a.batch = 1;
            const int c = i % copies;
            a.qweight = (const int32_t *)(q + (size_t)c * qwords); a.lookup_table = lut + (size_t)c * lutn; a.vec = x; a.mul = y + (size_t)i * N;
            if (sparse) { a.rows = rows + c * rstride; a.cols = cols + c * nstride; a.vals = vals + c * nstride; a.full_rows = fr + c * fstride; a.full_row_indices = fri; a.topX = 10; }
            int rc = sparse == 2 ? sqllm_lutgemv_fused(&a, xh, 1, (char *)yh + (size_t)i * N * 2, 1, nullptr, ws, wsb, st) : sqllm_lutgemv(&a, st);
            if (rc) { printf("error: %s\n", sqllm_last_error()); exit(1); }
        }
    };
    cudaGraphExec_t exec = nullptr;
    run_chain(false); CK(cudaStreamSynchronize(st));
    if (use_graph) {
        cudaGraph_t g;
        CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeGlobal));
        run_chain(true);
        CK(cudaStreamEndCapture(st, &g));
        CK(cudaGraphInstantiate(&exec, g, 0));
    }
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float best = 1e9f;
    for (int r = 0; r < 6; ++r) {
        // flush L2 between chains so that weights come from HBM
        CK(cudaMemsetAsync(q + (size_t)(copies - 1) * qwords, 0x5a, qwords * 4, st));
        CK(cudaEventRecord(e0, st));
        if (use_graph) CK(cudaGraphLaunch(exec, st)); else run_chain(true);
        CK(cudaEventRecord(e1, st)); CK(cudaStreamSynchronize(st));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); best = std::min(best, ms);
    }
    const int G = sqllm_debug_last_grid();
    printf("w%d %dx%d chain=%d graph=%d grid=%d : %.2f us per GEMV (best of 6 chains)\n", bits, K, N, chain, use_graph, G, best * 1e3 / chain);
    std::vector<unsigned long long> h(stride * chain);
    CK(cudaMemcpy(h.data(), trace, stride * 8 * chain, cudaMemcpyDeviceToHost));
    unsigned long long t00 = ~0ull;
    for (int c = 0; c < G; ++c) if (h[c * 32]) t00 = std::min(t00, h[c * 32]);
    const char *names[16] = {"entry", "sync0", "pre-wait", "post-wait", "x-staged", "1st-full", "loop-end", "sync1", "tma-1st", "tma-last", "sparse", "exit", "smid", "sp-prewait", "sp-postwait", "sp-hybdone"};
    printf("%-4s", "k");
    for (int s = 0; s < 16; ++s) if (s != 12) printf(" %9s(min/max)", names[s]);
    printf("\n");
    for (int i = 0; i < chain; ++i) {
        printf("%-4d", i);
        for (int s = 0; s < 16; ++s) {
            if (s == 12) continue;
            unsigned long long mn = ~0ull, mx = 0;
            for (int c = 0; c < G; ++c) { unsigned long long v = h[(size_t)i * stride + c * 32 + s]; if (v) { mn = std::min(mn, v); mx = std::max(mx, v); } }
            if (mx) printf(" %8.2f/%8.2f", (mn - t00) / 1e3, (mx - t00) / 1e3); else printf(" %17s", "-");
        }
        printf("\n");
    }
    {   // per-CTA detail of a steady-state launch, relative to that launch's min post-wait.  v2 marks: 16+s = table of segment s ready,
        // 24+s = segment s done; 8/9 = builders: polls through / y written; 10 = sparse warp 0 done
        const int i = chain - 2;
        unsigned long long base = ~0ull;
        for (int c = 0; c < G; ++c) { unsigned long long v = h[(size_t)i * stride + c * 32 + 3]; if (v) base = std::min(base, v); }
        printf("launch %d per-CTA (us rel. to min post-wait): cta smid entry post-wait x-staged | tab0 seg0 tab1 seg1 tab2 seg2 | loop-end sparse polls y-done exit\n", i);
        const int step = getenv("TRACE_ALL") ? 1 : (G > 64 ? 7 : 1);
        for (int c = 0; c < G; c += step) {
            const unsigned long long *r = &h[(size_t)i * stride + c * 32];
            auto rel = [&](unsigned long long v) { return v ? ((double)v - (double)base) / 1e3 : -99.0; };
            printf("%4d %4d %7.2f %6.2f %6.2f |", c, (int)r[12] - 1, rel(r[0]), rel(r[3]), rel(r[4]));
            for (int s2 = 0; s2 < 3; ++s2) printf(" %6.2f %6.2f", rel(r[16 + s2]), rel(r[24 + s2]));
            printf(" | %6.2f %6.2f %6.2f %6.2f %6.2f\n", rel(r[6]), rel(r[10]), rel(r[8]), rel(r[9]), rel(r[11]));
        }
    }
    return 0;
}
