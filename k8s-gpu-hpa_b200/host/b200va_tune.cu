// b200va_tune -- geometry / placement / ceiling experiments for the vectorAdd kernels, through
// the C ABI of the full-matrix library (libb200va_tune.so).
//
// Reads one geometry per line from stdin:
//     kind threads unroll ctas_per_sm ld_hint st_hint stages tile_bytes store_mode [early_loads [scheduler]]
// and prints one JSON line per geometry: bit-exactness (device-side recompute + digest against
// a K0 run), median / best per-launch time over P interleaved rounds of R back-to-back launches
// between two CUDA events, algorithmic GB/s (12 B/element).
//
//     b200va_tune [--n ELEMS] [--reps R] [--warmup W] [--rounds P]
//                 [--cold]        rotate through enough (A,B,C) sets that the footprint is >= 4x L2:
//                                 every launch streams from HBM (what the stager's chunks see)
//                 [--skew BYTES]  carve A, B, C out of ONE allocation with B at +BYTES and C at
//                                 +2*BYTES relative to their natural n*4 spacing (HBM channel phase)
//                 [--probes]      also time the ceiling probes (b200va_probe_f32) on the same buffers: read2
//                                 (two arrays in, nothing out), fill (one array out), copy (1 in 1 out)
//                 < geometries.txt
//
// Not part of the reference's surface: a development tool for geometry A/B runs.
#include <cuda_runtime.h>

#include <algorithm>
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b200va.h"

#define CK(expr)                                                                           \
    do {                                                                                   \
        cudaError_t e__ = (expr);                                                          \
        if (e__ != cudaSuccess) {                                                          \
            std::fprintf(stderr, "%s failed: %s\n", #expr, cudaGetErrorString(e__));       \
            std::exit(1);                                                                  \
        }                                                                                  \
    } while (0)

#define VA(expr)                                                                           \
    do {                                                                                   \
        int rc__ = (expr);                                                                 \
        if (rc__ != B200VA_OK) {                                                           \
            std::fprintf(stderr, "%s failed: %s (%d)\n", #expr, b200va_strerror(rc__), rc__); \
            std::exit(1);                                                                  \
        }                                                                                  \
    } while (0)

int main(int argc, char** argv)
{
    size_t n = size_t{1} << 28, skew = 0;
    int reps = 20, warmup = 3, rounds = 5;
    bool cold = false, probes = false;
    for (int i = 1; i < argc; ++i) {
        if (!std::strcmp(argv[i], "--n") && i + 1 < argc) n = std::strtoull(argv[++i], nullptr, 0);
        else if (!std::strcmp(argv[i], "--reps") && i + 1 < argc) reps = std::atoi(argv[++i]);
        else if (!std::strcmp(argv[i], "--warmup") && i + 1 < argc) warmup = std::atoi(argv[++i]);
        else if (!std::strcmp(argv[i], "--rounds") && i + 1 < argc) rounds = std::atoi(argv[++i]);
        else if (!std::strcmp(argv[i], "--skew") && i + 1 < argc) skew = std::strtoull(argv[++i], nullptr, 0);
        else if (!std::strcmp(argv[i], "--cold")) cold = true;
        else if (!std::strcmp(argv[i], "--probes")) probes = true;
        else {
            std::fprintf(stderr, "usage: %s [--n N] [--reps R] [--warmup W] [--rounds P] [--cold] [--skew BYTES] [--probes] < geometries\n", argv[0]);
            return 2;
        }
    }
    if (skew & 15u) { std::fprintf(stderr, "--skew must be a multiple of 16 bytes\n"); return 2; }
    b200va_devinfo_t di;
    VA(b200va_query(0, &di));
    CK(cudaSetDevice(0));

    // (A, B, C) sets carved from one allocation: set s at s*set_stride, B at +n*4+skew, C at +2*(n*4+skew)
    const size_t arr_bytes = n * sizeof(float);
    const size_t set_stride = (3 * (arr_bytes + skew) + 255) & ~size_t{255};
    const size_t want = cold ? 4 * static_cast<size_t>(di.l2_bytes) : 0;
    const int sets = static_cast<int>(std::max<size_t>(1, (want + 3 * arr_bytes - 1) / (3 * arr_bytes)));
    unsigned char* pool = nullptr;
    CK(cudaMalloc(&pool, static_cast<size_t>(sets) * set_stride + 256));
    auto A = [&](int s) { return reinterpret_cast<float*>(pool + static_cast<size_t>(s) * set_stride); };
    auto B = [&](int s) { return reinterpret_cast<float*>(pool + static_cast<size_t>(s) * set_stride + arr_bytes + skew); };
    auto C = [&](int s) { return reinterpret_cast<float*>(pool + static_cast<size_t>(s) * set_stride + 2 * (arr_bytes + skew)); };
    std::printf("{\"device\": \"%s\", \"sm_count\": %d, \"l2_bytes\": %d, \"n\": %zu, \"cold\": %s, \"buffer_sets\": %d, \"skew_bytes\": %zu}\n",
                di.name, di.sm_count, di.l2_bytes, n, cold ? "true" : "false", sets, skew);

    uint64_t *dRes, hRes[2], refDig[2];
    CK(cudaMalloc(&dRes, 2 * sizeof(uint64_t)));
    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    for (int s = 0; s < sets; ++s) {
        VA(b200va_fill_ctr_f32(A(s), n, 0x0A, 0, st));
        VA(b200va_fill_ctr_f32(B(s), n, 0x0B, 0, st));
    }

    // reference digest from the scalar control kernel
    VA(b200va_add_f32(A(0), B(0), C(0), n, B200VA_K0_SCALAR, st));
    VA(b200va_digest_f32(C(0), n, dRes, st));
    CK(cudaMemcpyAsync(refDig, dRes, sizeof refDig, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));

    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));

    // read every geometry, check each once for bit-exactness, then time them in `rounds`
    // interleaved passes (so drift hits all geometries alike).  One timing sample = `reps`
    // back-to-back launches between two events (no event inside the batch: the launches
    // chain through programmatic dependent launch exactly as in production).  With
    // early_loads = 1 the chain is legal: consecutive launches never write each other's inputs.
    struct Geo { b200va_tune_t t; unsigned long long bad = 0; bool dig_ok = false; std::string err; std::vector<double> ms; };
    std::vector<Geo> geos;
    char line[512];
    while (std::fgets(line, sizeof line, stdin)) {
        if (line[0] == '#' || line[0] == '\n') continue;
        Geo g{};
        b200va_tune_t& t = g.t;
        const int got = std::sscanf(line, "%d %d %d %d %d %d %d %d %d %d %d", &t.kind, &t.threads, &t.unroll, &t.ctas_per_sm,
                                    &t.ld_hint, &t.st_hint, &t.stages, &t.tile_bytes, &t.store_mode, &t.early_loads, &t.scheduler);
        if (got < 9) {
            std::fprintf(stderr, "bad geometry line: %s", line);
            continue;
        }
        geos.push_back(g);
    }
    for (auto& g : geos) {
        CK(cudaMemsetAsync(C(0), 0xff, n * sizeof(float), st));
        int rc = b200va_add_f32_tuned(A(0), B(0), C(0), n, &g.t, st);
        cudaError_t se = cudaStreamSynchronize(st);
        if (rc != B200VA_OK || se != cudaSuccess) {
            g.err = rc != B200VA_OK ? b200va_strerror(rc) : cudaGetErrorString(se);
            if (se != cudaSuccess) { std::fprintf(stderr, "sticky CUDA error: %s\n", g.err.c_str()); return 1; }
            continue;
        }
        VA(b200va_verify_f32(A(0), B(0), C(0), n, dRes, st));
        CK(cudaMemcpyAsync(hRes, dRes, sizeof hRes, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        g.bad = hRes[0];
        VA(b200va_digest_f32(C(0), n, dRes, st));
        CK(cudaMemcpyAsync(hRes, dRes, sizeof hRes, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        g.dig_ok = hRes[0] == refDig[0] && hRes[1] == refDig[1];
    }
    auto time_batch = [&](auto&& launch_one) {
        for (int i = 0; i < warmup; ++i) launch_one(i % sets);
        CK(cudaEventRecord(e0, st));
        for (int i = 0; i < reps; ++i) launch_one((warmup + i) % sets);
        CK(cudaEventRecord(e1, st));
        CK(cudaStreamSynchronize(st));
        float total = 0.f;
        CK(cudaEventElapsedTime(&total, e0, e1));
        return static_cast<double>(total) / reps;
    };
    std::vector<double> p_read, p_fill, p_copy;
    for (int r = 0; r < rounds; ++r) {
        for (auto& g : geos) {
            if (!g.err.empty()) continue;
            g.ms.push_back(time_batch([&](int s) { VA(b200va_add_f32_tuned(A(s), B(s), C(s), n, &g.t, st)); }));
        }
        if (probes) {
            p_read.push_back(time_batch([&](int s) { VA(b200va_probe_f32(B200VA_PROBE_READ2, A(s), B(s), C(s), n, st)); }));
            p_fill.push_back(time_batch([&](int s) { VA(b200va_probe_f32(B200VA_PROBE_FILL, nullptr, nullptr, C(s), n, st)); }));
            p_copy.push_back(time_batch([&](int s) { VA(b200va_probe_f32(B200VA_PROBE_COPY, A(s), nullptr, C(s), n, st)); }));
        }
    }
    const double bytes = 12.0 * static_cast<double>(n);
    for (auto& g : geos) {
        const b200va_tune_t& t = g.t;
        std::printf("{\"kind\": %d, \"threads\": %d, \"unroll\": %d, \"ctas_per_sm\": %d, \"ld\": %d, \"st\": %d, "
                    "\"stages\": %d, \"tile_bytes\": %d, \"store_mode\": %d, \"early\": %d, \"sched\": %d, ", t.kind, t.threads, t.unroll,
                    t.ctas_per_sm, t.ld_hint, t.st_hint, t.stages, t.tile_bytes, t.store_mode, t.early_loads, t.scheduler);
        if (!g.err.empty()) { std::printf("\"error\": \"%s\"}\n", g.err.c_str()); continue; }
        std::sort(g.ms.begin(), g.ms.end());
        double mean = 0;
        for (double v : g.ms) mean += v;
        mean /= static_cast<double>(g.ms.size());
        const double med = g.ms[g.ms.size() / 2], best = g.ms[0];
        std::printf("\"mismatches\": %llu, \"digest_ok\": %s, \"samples\": %zu, \"launches_per_sample\": %d, "
                    "\"ms_median\": %.5f, \"ms_best\": %.5f, \"ms_mean\": %.5f, \"GBps_median\": %.1f, "
                    "\"GBps_best\": %.1f, \"GBps_mean\": %.1f, \"elems_per_s\": %.4e}\n",
                    g.bad, g.dig_ok ? "true" : "false", g.ms.size(), reps, med, best, mean, bytes / med / 1e6,
                    bytes / best / 1e6, bytes / mean / 1e6, static_cast<double>(n) / (med * 1e-3));
    }
    auto report_probe = [&](const char* name, std::vector<double>& ms, double bytes_per_elem, const char* what) {
        if (ms.empty()) return;
        std::sort(ms.begin(), ms.end());
        const double med = ms[ms.size() / 2];
        std::printf("{\"probe\": \"%s\", \"what\": \"%s\", \"bytes_per_element\": %.0f, \"ms_median\": %.5f, \"ms_best\": %.5f, "
                    "\"GBps_median\": %.1f, \"GBps_best\": %.1f}\n", name, what, bytes_per_elem, med, ms[0],
                    bytes_per_elem * static_cast<double>(n) / med / 1e6, bytes_per_elem * static_cast<double>(n) / ms[0] / 1e6);
    };
    report_probe("read2", p_read, 8, "load A and B (128-bit, 512 thr x 1), store nothing");
    report_probe("fill", p_fill, 4, "store C (128-bit, L1::no_allocate), load nothing");
    report_probe("copy", p_copy, 8, "C = A (1 read : 1 write)");
    return 0;
}
