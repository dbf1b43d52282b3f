// seq_trace.cu - timing and per-CTA timeline of the sequence kernel (C ABI) on LLaMA-shaped decoder layers with synthetic buffers.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a [-DSQLLM_TRACE] -I include -o tests/perf/seq_trace tests/perf/seq_trace.cu squeezellm_b200/csrc/*.cu
//   ./seq_trace bits hidden ffn layers lut_mode(0|1) sparse(0|1) [trace_layer]
// Prints us per token and per decoder layer; with -DSQLLM_TRACE also, for the 4 GEMVs of `trace_layer`, min / median / max over CTAs of
// every phase stamp relative to the first stamp of that layer.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "sqllm_b200.h"
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

struct Mat { int K, N; uint32_t *q; float *lut; int *rows, *cols; float *vals, *fr; int *fri; };

static Mat make(int bits, int K, int N, int sparse) {
    Mat m; memset(&m, 0, sizeof(m)); m.K = K; m.N = N;
    const size_t qwords = (size_t)K / 32 * bits * N;
    CK(cudaMalloc(&m.q, qwords * 4)); CK(cudaMemset(m.q, 0x5a, qwords * 4));
    CK(cudaMalloc(&m.lut, (size_t)N * 16 * 4)); CK(cudaMemset(m.lut, 0, (size_t)N * 16 * 4));
    if (sparse) {
        const int per = (int)(0.0045 * K + 0.5); const size_t nnz = (size_t)per * N;
        std::vector<int> hr(N + 1), hc(nnz);
        for (int c = 0; c <= N; ++c) hr[c] = c * per;
        for (size_t i = 0; i < nnz; ++i) hc[i] = (int)((i * 2654435761u) % K);
        CK(cudaMalloc(&m.rows, (N + 1) * 4)); CK(cudaMalloc(&m.cols, nnz * 4)); CK(cudaMalloc(&m.vals, nnz * 4));
        CK(cudaMemset(m.vals, 0, nnz * 4));
        CK(cudaMemcpy(m.rows, hr.data(), (N + 1) * 4, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(m.cols, hc.data(), nnz * 4, cudaMemcpyHostToDevice));
        CK(cudaMalloc(&m.fr, (size_t)K * 10 * 4)); CK(cudaMemset(m.fr, 0, (size_t)K * 10 * 4));
        CK(cudaMalloc(&m.fri, 40)); CK(cudaMemset(m.fri, 0, 40));
    }
    return m;
}

int main(int argc, char **argv) {
    setvbuf(stdout, NULL, _IONBF, 0);
    const int bits = argc > 1 ? atoi(argv[1]) : 4, H = argc > 2 ? atoi(argv[2]) : 4096, F = argc > 3 ? atoi(argv[3]) : 11008;
    const int layers = argc > 4 ? atoi(argv[4]) : 8, mode = argc > 5 ? atoi(argv[5]) : 0, sparse = argc > 6 ? atoi(argv[6]) : 1;
    const int tl = argc > 7 ? atoi(argv[7]) : layers / 2;
    std::vector<sqllm_seq_item> items;
    void *x; CK(cudaMalloc(&x, H * 2)); CK(cudaMemset(x, 0, H * 2));
    const int dims[4][3] = {{H, 3 * H, 0}, {H, H, 2 * H}, {H, 2 * F, 0}, {F, H, 0}};
    for (int l = 0; l < layers; ++l)
        for (int j = 0; j < 4; ++j) {
            Mat m = make(bits, dims[j][0], dims[j][1], sparse);
            sqllm_seq_item it; memset(&it, 0, sizeof(it));
            it.a.bits = bits; it.a.in_features = m.K; it.a.out_features = m.N; it.a.batch = 1;
            it.a.qweight = (const int32_t *)m.q; it.a.lookup_table = m.lut;
            if (sparse) { it.a.rows = m.rows; it.a.cols = m.cols; it.a.vals = m.vals; it.a.full_rows = m.fr; it.a.full_row_indices = m.fri; it.a.topX = 10; }
            it.x_from = (int)items.size() - 1; it.x_offset = dims[j][2];
            if (items.empty()) { it.x_from = -1; it.x_ext = x; }
            it.members = 1; it.out_features_full = m.N;
            items.push_back(it);
        }
    const int n = (int)items.size();
    uint64_t *trace = nullptr;
#ifdef SQLLM_TRACE
    CK(cudaMalloc(&trace, (size_t)n * 1024 * 32 * 8)); CK(cudaMemset(trace, 0, (size_t)n * 1024 * 32 * 8));
#endif
    void *ydst; CK(cudaMalloc(&ydst, H * 2));
    int ex_item = n - 1; void *ex_dst = ydst;
    sqllm_seq_options o; memset(&o, 0, sizeof(o));
    o.lut_mode = mode; o.world = 1; o.n_export = 1; o.export_items = &ex_item; o.export_dst = &ex_dst; o.trace = trace;
    sqllm_sequence *s = nullptr;
    if (sqllm_sequence_create(items.data(), n, &o, &s)) { printf("create: %s\n", sqllm_last_error()); return 1; }
    cudaStream_t st; CK(cudaStreamCreate(&st));
    for (int i = 0; i < 3; ++i) if (sqllm_sequence_run(s, st)) { printf("run: %s\n", sqllm_last_error()); return 1; }
    CK(cudaStreamSynchronize(st));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    const int reps = 20;
    CK(cudaEventRecord(e0, st));
    for (int i = 0; i < reps; ++i) sqllm_sequence_run(s, st);
    CK(cudaEventRecord(e1, st)); CK(cudaStreamSynchronize(st));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    printf("w%d hidden=%d ffn=%d layers=%d mode=%s sparse=%d : %.1f us per token, %.2f us per decoder layer (err=%d)\n", bits, H, F, layers,
           mode ? "fp16" : "exact", sparse, ms * 1e3 / reps, ms * 1e3 / reps / layers, sqllm_sequence_error(s, st));
#ifdef SQLLM_TRACE
    std::vector<uint64_t> h((size_t)n * 1024 * 32);
    CK(cudaMemcpy(h.data(), trace, h.size() * 8, cudaMemcpyDeviceToHost));
    const int G = sqllm_device_sm_count();
    uint64_t t00 = ~0ull;
    for (int c = 0; c < G; ++c) { uint64_t v = h[((size_t)(4 * tl) * 1024 + c) * 32 + 2]; if (v) t00 = std::min(t00, v); }
    const int slots[] = {2, 4, 16, 24, 17, 25, 6, 10, 12, 13, 14, 15, 8, 9};
    const char *names[] = {"top", "x-staged", "tab0", "seg0-done", "tab1", "seg1-done", "loop-end", "sparse", "b-tabs", "b-flushed", "b-acc", "b-cbox", "fin-polls", "y-done"};
    printf("layer %d, us relative to its first stamp; min / median / max over CTAs\n%-4s", tl, "gemv");
    for (auto nm : names) printf(" %22s", nm);
    printf("\n");
    for (int g = 4 * tl; g < 4 * tl + 5 && g < n; ++g) {
        printf("%-4d", g);
        for (int sl : slots) {
            std::vector<double> v;
            for (int c = 0; c < G; ++c) { uint64_t t = h[((size_t)g * 1024 + c) * 32 + sl]; if (t) v.push_back(((double)t - (double)t00) / 1e3); }
            if (v.empty()) { printf(" %22s", "-"); continue; }
            std::sort(v.begin(), v.end());
            printf("  %6.2f/%6.2f/%6.2f", v.front(), v[v.size() / 2], v.back());
        }
        printf("\n");
    }
    // per-CTA rows of the CTAs that finish a GEMV last (by y-done), and of the first / a middle one for comparison
    for (int g = 4 * tl; g < 4 * tl + 4 && g < n; ++g) {
        std::vector<std::pair<double, int>> order;
        for (int c = 0; c < G; ++c) { uint64_t t = h[((size_t)g * 1024 + c) * 32 + 9]; if (t) order.push_back({((double)t - (double)t00) / 1e3, c}); }
        std::sort(order.begin(), order.end());
        printf("gemv %d: latest CTAs by y-done | cta:", g);
        for (auto nm : names) printf(" %9s", nm);
        printf("\n");
        std::vector<int> pick;
        for (int i = 0; i < 6 && i < (int)order.size(); ++i) pick.push_back(order[order.size() - 1 - i].second);
        if (!order.empty()) { pick.push_back(order[0].second); pick.push_back(order[order.size() / 2].second); }
        for (int c : pick) {
            printf("   %4d:", c);
            for (int sl : slots) { uint64_t t = h[((size_t)g * 1024 + c) * 32 + sl]; if (t) printf(" %9.2f", ((double)t - (double)t00) / 1e3); else printf(" %9s", "-"); }
            printf("\n");
        }
    }
#endif
    sqllm_sequence_destroy(s);
    return 0;
}
