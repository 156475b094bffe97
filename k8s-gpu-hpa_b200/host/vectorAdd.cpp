// vectorAdd -- the H100-native replacement for the binary the reference runs as
//
//     image:   "k8s.gcr.io/cuda-vector-add:v0.1"                     cuda-test-deployment.yaml:18
//     command: for (( c=1; c<=5000; c++ )); do ./vectorAdd; done     cuda-test-deployment.yaml:19
//
// Outer drop-in boundary = this process.  With NO arguments it behaves like the image's
// binary (SURVEY.md section 8(a), rows a2-a7): 50000 fp32 elements filled with the
// never-seeded rand() recipe, copied to the GPU, added once, copied back, verified,
// "Test PASSED" / "Done", exit 0 -- so the unchanged bash loop of the Deployment drives
// it.  Verification is stricter than the sample's 1e-5: bitwise.
// Any failure prints to stderr and exits 1 (the sample's convention).  There is no CPU
// fallback: without a GPU the process fails.
//
// Options move the reference's *bash* loop count in-process and add the benchmark
// shapes of BASELINE.json:
//   --n N            elements (default 50000)            --iters K   launches (default 1)
//   --gpus G         shard [0,N) evenly over G GPUs      --kernel auto|k0|k1|k2|k3
//   --mode sample|resident|staged                        --gen rand|ctr
//   --graph B        capture B launches per CUDA graph   --verify full|none
//   --seed S         ctr generator seeds: A = S, B = S+1 (default 0x0A)
//   --duration S     repeat the K-launch block for S seconds of wall clock
//   --target-util P  duty-cycle the blocks so the GPU is busy ~P % of each period
//   --period-ms M    duty-cycle period (default 100)     --nvml  sample NVML utilisation
//   --hpa-threshold T  utilisation the HPA compares with (default 5, cuda-test-hpa.yaml:21)
//   --cpu-baseline   also time a host-threads C[i]=A[i]+B[i] loop (reported, never used)
//   --json PATH      write the result line to PATH as well as stdout
//   --metrics-file P rewrite P every 0.5 s with `dcgm_gpu_utilization{...} <NVML util>` (Prometheus text;
//                    the namespace label comes from $POD_NAMESPACE, default "default")
//   --host-mem pinned|pageable   staged mode: library-allocated pinned arrays (default) or plain malloc,
//                    what the reference process has; the stager page-locks those once and reuses them
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <sched.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cinttypes>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/b200va.h"

namespace {

using clk = std::chrono::steady_clock;

double secs_since(clk::time_point t0) { return std::chrono::duration<double>(clk::now() - t0).count(); }

[[noreturn]] void die(const char* what, const char* why)
{
    std::fprintf(stderr, "Failed to %s (error code %s)!\n", what, why);
    std::exit(EXIT_FAILURE);
}

void ck(cudaError_t e, const char* what)
{
    if (e != cudaSuccess) die(what, cudaGetErrorString(e));
}

void va(int rc, const char* what)
{
    if (rc != B200VA_OK) die(what, b200va_strerror(rc));
}

struct Options {
    size_t n = 50000;
    int iters = 1;
    int gpus = 1;
    int variant = B200VA_K_AUTO;
    std::string mode = "sample";
    std::string gen = "rand";
    bool gen_set = false, mode_set = false;
    int graph = 0;
    bool verify = true;
    double duration = 0.0;
    double target_util = 0.0;
    double period_ms = 100.0;
    bool nvml = false;
    double hpa_threshold = 5.0;
    bool cpu_baseline = false;
    int cpu_threads = 0;
    uint64_t seed = 0x0A;        // ctr generator: A uses seed, B uses seed + 1 (defaults 0x0A / 0x0B)
    int stage_mode = B200VA_STAGE_AUTO;   // staged mode pipeline: auto (lanes / register-once), 0 slot streams, 1 zero-copy
    bool pageable = false;       // staged mode: host arrays from plain malloc instead of b200va_host_alloc
    std::string json_path;
    std::string metrics_file;    // Prometheus text snapshot of the NVML utilisation (GPU 0), rewritten every 0.5 s
    bool any = false;
};

int host_cpus()
{
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof set, &set) == 0 && CPU_COUNT(&set) > 0) return CPU_COUNT(&set);
    const long c = sysconf(_SC_NPROCESSORS_ONLN);
    return c > 0 ? static_cast<int>(c) : 1;
}

// Container CPU bandwidth quota in CPUs (cgroup v2 cpu.max), 0 if unlimited/unknown.
double cpu_quota()
{
    FILE* f = std::fopen("/sys/fs/cgroup/cpu.max", "r");
    if (!f) return 0.0;
    char q[64];
    double period = 0;
    const int got = std::fscanf(f, "%63s %lf", q, &period);
    std::fclose(f);
    return (got == 2 && std::strcmp(q, "max") != 0 && period > 0) ? std::atof(q) / period : 0.0;
}

int parse_variant(const char* s)
{
    if (!std::strcmp(s, "auto")) return B200VA_K_AUTO;
    if (!std::strcmp(s, "k0")) return B200VA_K0_SCALAR;
    if (!std::strcmp(s, "k1")) return B200VA_K1_VEC128;
    if (!std::strcmp(s, "k2")) return B200VA_K2_TMA;
    if (!std::strcmp(s, "k3")) return B200VA_K3_VEC256;
    std::fprintf(stderr, "unknown --kernel %s (auto|k0|k1|k2|k3)\n", s);
    std::exit(EXIT_FAILURE);
}

const char* variant_name(int v)
{
    switch (v) {
        case B200VA_K0_SCALAR: return "k0_scalar";
        case B200VA_K1_VEC128: return "k1_vec128";
        case B200VA_K2_TMA: return "k2_tma";
        case B200VA_K3_VEC256: return "k3_vec256";
    }
    return "auto";
}

size_t parse_size(const char* s)
{
    // accepts 268435456, 2^28, 1<<28
    const char* p = std::strchr(s, '^');
    if (p) return static_cast<size_t>(std::pow(std::strtod(s, nullptr), std::strtod(p + 1, nullptr)) + 0.5);
    p = std::strstr(s, "<<");
    if (p) return static_cast<size_t>(std::strtoull(s, nullptr, 0)) << std::strtoul(p + 2, nullptr, 0);
    return static_cast<size_t>(std::strtoull(s, nullptr, 0));
}

Options parse(int argc, char** argv)
{
    Options o;
    auto need = [&](int& i) -> const char* {
        if (i + 1 >= argc) { std::fprintf(stderr, "%s needs a value\n", argv[i]); std::exit(EXIT_FAILURE); }
        return argv[++i];
    };
    for (int i = 1; i < argc; ++i) {
        const std::string a = argv[i];
        o.any = true;
        if (a == "--n") o.n = parse_size(need(i));
        else if (a == "--iters") o.iters = std::atoi(need(i));
        else if (a == "--gpus") o.gpus = std::atoi(need(i));
        else if (a == "--kernel") o.variant = parse_variant(need(i));
        else if (a == "--mode") { o.mode = need(i); o.mode_set = true; }
        else if (a == "--gen") { o.gen = need(i); o.gen_set = true; }
        else if (a == "--graph") o.graph = std::atoi(need(i));
        else if (a == "--seed") o.seed = std::strtoull(need(i), nullptr, 0);
        else if (a == "--verify") o.verify = std::strcmp(need(i), "none") != 0;
        else if (a == "--duration") o.duration = std::atof(need(i));
        else if (a == "--target-util") o.target_util = std::atof(need(i));
        else if (a == "--period-ms") o.period_ms = std::atof(need(i));
        else if (a == "--nvml") o.nvml = true;
        else if (a == "--hpa-threshold") o.hpa_threshold = std::atof(need(i));
        else if (a == "--cpu-baseline") o.cpu_baseline = true;
        else if (a == "--cpu-threads") o.cpu_threads = std::atoi(need(i));
        else if (a == "--zero-copy") o.stage_mode = B200VA_STAGE_ZEROCOPY;
        else if (a == "--slot-streams") o.stage_mode = B200VA_STAGE_SLOTS;
        else if (a == "--bounce") o.stage_mode = B200VA_STAGE_BOUNCE;
        else if (a == "--host-mem") {
            const std::string v = need(i);
            if (v != "pinned" && v != "pageable") { std::fprintf(stderr, "bad --host-mem (pinned|pageable)\n"); std::exit(EXIT_FAILURE); }
            o.pageable = v == "pageable";
        }
        else if (a == "--json") o.json_path = need(i);
        else if (a == "--metrics-file") { o.metrics_file = need(i); o.nvml = true; }
        else if (a == "--help" || a == "-h") {
            std::printf("usage: vectorAdd [--n N] [--iters K] [--gpus G] [--kernel auto|k0|k1|k2|k3]\n"
                        "                 [--mode sample|resident|staged] [--gen rand|ctr] [--seed S] [--graph B]\n"
                        "                 [--verify full|none] [--duration S] [--target-util P] [--period-ms M]\n"
                        "                 [--nvml] [--hpa-threshold T] [--cpu-baseline] [--cpu-threads T]\n"
                        "                 [--zero-copy] [--host-mem pinned|pageable] [--json PATH] [--metrics-file PATH]\n"
                        "no arguments: the reference image's behaviour (50000 elements, one add, verify).\n");
            std::exit(0);
        } else {
            std::fprintf(stderr, "unknown option %s (try --help)\n", a.c_str());
            std::exit(EXIT_FAILURE);
        }
    }
    if (o.iters < 1 || o.gpus < 1 || o.graph < 0) { std::fprintf(stderr, "bad --iters/--gpus/--graph\n"); std::exit(EXIT_FAILURE); }
    if (!o.mode_set && (o.gpus > 1 || o.duration > 0 || o.target_util > 0)) o.mode = "resident";
    if (!o.gen_set) o.gen = (o.mode == "sample") ? "rand" : "ctr";
    if (o.mode != "sample" && o.mode != "resident" && o.mode != "staged") { std::fprintf(stderr, "bad --mode\n"); std::exit(EXIT_FAILURE); }
    if (o.gen != "rand" && o.gen != "ctr") { std::fprintf(stderr, "bad --gen\n"); std::exit(EXIT_FAILURE); }
    if (o.mode != "sample" && o.gen == "rand") { std::fprintf(stderr, "--gen rand needs --mode sample\n"); std::exit(EXIT_FAILURE); }
    if (o.mode == "sample" && o.gpus != 1) { std::fprintf(stderr, "--mode sample is single-GPU\n"); std::exit(EXIT_FAILURE); }
    return o;
}

// ------------------------------------------------------------------ host helpers
template <class F>
void parallel_spans(size_t n, int threads, F&& f)
{
    if (threads < 1) threads = 1;
    size_t chunk = (n + static_cast<size_t>(threads) - 1) / static_cast<size_t>(threads);
    chunk = (chunk + 15) & ~size_t{15};
    std::vector<std::thread> th;
    for (int t = 0; t < threads; ++t) {
        const size_t lo = std::min(n, static_cast<size_t>(t) * chunk), hi = std::min(n, lo + chunk);
        if (lo >= hi) break;
        th.emplace_back([&f, lo, hi] { f(lo, hi); });
    }
    for (auto& x : th) x.join();
}

// Reported baseline only (--cpu-baseline): a threaded host loop, timed; its output is
// discarded and never feeds the GPU result.
struct CpuBaseline { double elems_per_s = 0, gbps = 0, ms_median = 0; int threads = 0; size_t n = 0; };

CpuBaseline run_cpu_baseline(size_t n, int threads)
{
    CpuBaseline r;
    if (threads <= 0) {   // more runnable threads than ~2x the cgroup quota only get throttled
        threads = host_cpus();
        const double q = cpu_quota();
        if (q > 0) threads = std::max(1, std::min(threads, static_cast<int>(2 * q + 0.5)));
    }
    r.threads = threads;
    r.n = n;
    float *a = nullptr, *b = nullptr, *c = nullptr;
    if (posix_memalign(reinterpret_cast<void**>(&a), 64, n * 4 + 64) || posix_memalign(reinterpret_cast<void**>(&b), 64, n * 4 + 64) ||
        posix_memalign(reinterpret_cast<void**>(&c), 64, n * 4 + 64))
        die("allocate CPU baseline vectors", "out of memory");
    parallel_spans(n, threads, [&](size_t lo, size_t hi) {   // first touch by the adding thread
        b200va_host_fill_ctr_f32(a + lo, hi - lo, 0x0A, lo);
        b200va_host_fill_ctr_f32(b + lo, hi - lo, 0x0B, lo);
        std::memset(c + lo, 0, (hi - lo) * 4);
    });
    std::vector<double> t;
    for (int rep = 0; rep < 6; ++rep) {
        const auto t0 = clk::now();
        parallel_spans(n, threads, [&](size_t lo, size_t hi) {
            for (size_t i = lo; i < hi; ++i) c[i] = a[i] + b[i];
        });
        if (rep) t.push_back(secs_since(t0));
    }
    std::sort(t.begin(), t.end());
    r.ms_median = t[t.size() / 2] * 1e3;
    r.elems_per_s = static_cast<double>(n) / t[t.size() / 2];
    r.gbps = 12.0 * static_cast<double>(n) / t[t.size() / 2] / 1e9;
    volatile float sink = c[n / 2];
    (void)sink;
    std::free(a); std::free(b); std::free(c);
    return r;
}

// ------------------------------------------------------------------ NVML (dlopen)
struct Nvml {
    using init_t = int (*)();
    using shut_t = int (*)();
    using byid_t = int (*)(const char*, void**);
    struct Util { unsigned gpu, memory; };
    using util_t = int (*)(void*, Util*);
    using uuid_t = int (*)(void*, char*, unsigned);
    void* lib = nullptr;
    shut_t shut = nullptr;
    util_t util = nullptr;
    std::vector<void*> dev;
    std::vector<std::string> uuid;
    bool open(const std::vector<int>& cuda_devs)
    {
        lib = dlopen("libnvidia-ml.so.1", RTLD_NOW);
        if (!lib) return false;
        auto init = reinterpret_cast<init_t>(dlsym(lib, "nvmlInit_v2"));
        shut = reinterpret_cast<shut_t>(dlsym(lib, "nvmlShutdown"));
        auto byid = reinterpret_cast<byid_t>(dlsym(lib, "nvmlDeviceGetHandleByPciBusId_v2"));
        util = reinterpret_cast<util_t>(dlsym(lib, "nvmlDeviceGetUtilizationRates"));
        if (!init || !shut || !byid || !util || init() != 0) return false;
        for (int d : cuda_devs) {
            char bus[32];
            void* h = nullptr;
            if (cudaDeviceGetPCIBusId(bus, sizeof bus, d) != cudaSuccess || byid(bus, &h) != 0) return false;
            dev.push_back(h);
            char id[96] = "unknown";
            if (auto get_uuid = reinterpret_cast<uuid_t>(dlsym(lib, "nvmlDeviceGetUUID"))) get_uuid(h, id, sizeof id);
            uuid.emplace_back(id);
        }
        return true;
    }
    // One sample in the Prometheus text format under the metric name the reference's rule reads
    // (cuda-test-prometheusrule.yaml:13), e.g. for node-exporter's textfile collector.  Written
    // atomically (tmp + rename).  The pod label is what the rule joins on.
    void write_metrics(const std::string& path, size_t i, int util_pct) const
    {
        const char* pod = std::getenv("HOSTNAME");
        const char* ns = std::getenv("POD_NAMESPACE");       // downward-API convention; the reference deploys into "default"
        const std::string tmp = path + ".tmp";
        if (FILE* f = std::fopen(tmp.c_str(), "w")) {
            std::fprintf(f, "# HELP dcgm_gpu_utilization GPU utilization (in %%), NVML utilization.gpu as sampled by vectorAdd.\n"
                            "# TYPE dcgm_gpu_utilization gauge\n"
                            "dcgm_gpu_utilization{gpu=\"%zu\",uuid=\"%s\",pod=\"%s\",namespace=\"%s\"} %d\n",
                         i, i < uuid.size() ? uuid[i].c_str() : "unknown", pod ? pod : "", (ns && *ns) ? ns : "default", util_pct);
            std::fclose(f);
            std::rename(tmp.c_str(), path.c_str());
        }
    }
    int gpu_util(size_t i) const
    {
        Util u{};
        return (i < dev.size() && util(dev[i], &u) == 0) ? static_cast<int>(u.gpu) : -1;
    }
    ~Nvml() { if (lib && shut) shut(); }
};

// B200VA_TRACE_STARTUP=1: milliseconds since process start at each step of the sample flow, on stderr
// (where does one ./vectorAdd process of the reference's 5000-process loop spend its time?).
struct StartupTrace {
    const bool on = [] { const char* e = std::getenv("B200VA_TRACE_STARTUP"); return e && e[0] == '1'; }();
    const clk::time_point t0 = clk::now();
    void mark(const char* what) const { if (on) std::fprintf(stderr, "[startup] %-28s %9.3f ms\n", what, secs_since(t0) * 1e3); }
};

// ------------------------------------------------------------------ sample mode (a2..a7)
int run_sample(const Options& o)
{
    const StartupTrace trace;
    const size_t n = o.n;
    const size_t size = n * sizeof(float);
    std::printf("[Vector addition of %zu elements]\n", n);

    float* h_A = static_cast<float*>(std::malloc(size ? size : 4));
    float* h_B = static_cast<float*>(std::malloc(size ? size : 4));
    float* h_C = static_cast<float*>(std::malloc(size ? size : 4));
    if (!h_A || !h_B || !h_C) {
        std::fprintf(stderr, "Failed to allocate host vectors!\n");
        return EXIT_FAILURE;
    }
    if (o.gen == "rand") {
        va(b200va_host_fill_rand_f32(h_A, h_B, n), "initialize host vectors");
    } else {
        parallel_spans(n, host_cpus(), [&](size_t lo, size_t hi) {
            b200va_host_fill_ctr_f32(h_A + lo, hi - lo, o.seed, lo);
            b200va_host_fill_ctr_f32(h_B + lo, hi - lo, o.seed + 1, lo);
        });
    }

    trace.mark("host vectors filled");
    float *d_A = nullptr, *d_B = nullptr, *d_C = nullptr;
    ck(cudaMalloc(&d_A, size ? size : 4), "allocate device vector A");
    trace.mark("first cudaMalloc (context)");
    ck(cudaMalloc(&d_B, size ? size : 4), "allocate device vector B");
    ck(cudaMalloc(&d_C, size ? size : 4), "allocate device vector C");

    std::printf("Copy input data from the host memory to the CUDA device\n");
    ck(cudaMemcpy(d_A, h_A, size, cudaMemcpyHostToDevice), "copy vector A from host to device");
    ck(cudaMemcpy(d_B, h_B, size, cudaMemcpyHostToDevice), "copy vector B from host to device");

    b200va_tune_t tune;
    unsigned grid = 0, block = 0;
    va(b200va_resolve(o.variant, n, &tune), "resolve kernel geometry");
    va(b200va_geometry(&tune, n, 0, &grid, &block, nullptr), "resolve kernel geometry");
    trace.mark("H2D copies done");
    std::printf("CUDA kernel launch with %u blocks of %u threads\n", grid, block);
    cudaStream_t st;
    ck(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking), "create stream");
    va(b200va_add_f32_loop(d_A, d_B, d_C, n, o.variant, o.iters, o.graph, st), "launch vectorAdd kernel");
    ck(cudaStreamSynchronize(st), "launch vectorAdd kernel");

    trace.mark("kernel(s) done");
    std::printf("Copy output data from the CUDA device to the host memory\n");
    ck(cudaMemcpy(h_C, d_C, size, cudaMemcpyDeviceToHost), "copy vector C from device to host");

    if (o.verify) {
        size_t bad = 0;
        if (b200va_host_verify_f32(h_A, h_B, h_C, n, &bad) != B200VA_OK) {
            std::fprintf(stderr, "Result verification failed at element %zu!\n", bad);
            return EXIT_FAILURE;
        }
        std::printf("Test PASSED\n");
    } else {
        std::printf("Test SKIPPED (--verify none)\n");   // never claim a pass that was not checked
    }

    trace.mark("D2H + verify done");
    ck(cudaStreamDestroy(st), "destroy stream");
    ck(cudaFree(d_A), "free device vector A");
    ck(cudaFree(d_B), "free device vector B");
    ck(cudaFree(d_C), "free device vector C");
    std::free(h_A); std::free(h_B); std::free(h_C);
    trace.mark("device memory freed");
    ck(cudaDeviceReset(), "deinitialize the device");
    trace.mark("cudaDeviceReset done");
    std::printf("Done\n");
    return EXIT_SUCCESS;
}

// ------------------------------------------------------------------ sharded modes
struct Barrier {
    std::mutex m; std::condition_variable cv; int count, waiting = 0, gen = 0;
    explicit Barrier(int c) : count(c) {}
    void wait()
    {
        std::unique_lock<std::mutex> lk(m);
        const int g = gen;
        if (++waiting == count) { waiting = 0; ++gen; cv.notify_all(); }
        else cv.wait(lk, [&] { return g != gen; });
    }
};

struct ShardResult {
    size_t begin = 0, end = 0;
    double gpu_ms = 0;          // sum of event-timed kernel blocks
    double wall_s = 0;
    long long launches = 0;
    uint64_t mismatches = 0, first_bad = ~0ull, digest[2] = {0, 0};
    std::vector<int> util_samples;
    double first_pass_wall_ms = 0;   // staged: wall clock of the first pass (register-once pays its pinning here)
    int stage_mode = -2;             // staged: the pipeline the stager resolved to on the last pass
    int first_stage_mode = -2;       // ... and on the first (4 = it page-locked the arrays; later passes then see pinned memory: 2)
    std::string error;
};

void shard_worker(const Options& o, int rank, Barrier& bar, ShardResult& r, Nvml* nvml)
{
    auto fail = [&](const char* what, const char* why) { r.error = std::string(what) + ": " + why; };
    size_t b = 0, e = 0;
    b200va_shard_range(o.n, o.gpus, rank, &b, &e);
    r.begin = b; r.end = e;
    const size_t m = e - b;
    bool ok = true;
    auto CK = [&](cudaError_t err, const char* what) { if (ok && err != cudaSuccess) { fail(what, cudaGetErrorString(err)); ok = false; } };
    auto VA = [&](int rc, const char* what) {
        if (ok && rc != B200VA_OK) { fail(what, (std::string(b200va_strerror(rc)) + " [" + std::to_string(rc) + "]").c_str()); ok = false; }
    };

    CK(cudaSetDevice(rank), "select device");
    float *dA = nullptr, *dB = nullptr, *dC = nullptr, *hA = nullptr, *hB = nullptr, *hC = nullptr;
    uint64_t* dRes = nullptr;
    cudaStream_t st = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    b200va_stager_t* stager = nullptr;
    b200va_loop_t* loop = nullptr;
    const bool staged = o.mode == "staged";
    if (ok) {
        CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking), "create stream");
        CK(cudaEventCreate(&e0), "create event"); CK(cudaEventCreate(&e1), "create event");
        CK(cudaMalloc(&dRes, 4 * sizeof(uint64_t)), "allocate result words");
        if (staged) {
            if (o.pageable) {
                // the reference process's own memory: plain malloc (a2); the stager page-locks it on first sight
                hA = static_cast<float*>(std::malloc(m ? m * 4 : 4));
                hB = static_cast<float*>(std::malloc(m ? m * 4 : 4));
                hC = static_cast<float*>(std::malloc(m ? m * 4 : 4));
                if (!hA || !hB || !hC) { fail("allocate host vectors", "out of memory"); ok = false; }
            } else {
                VA(b200va_host_alloc(reinterpret_cast<void**>(&hA), m * 4), "allocate pinned A");
                VA(b200va_host_alloc(reinterpret_cast<void**>(&hB), m * 4), "allocate pinned B");
                VA(b200va_host_alloc(reinterpret_cast<void**>(&hC), m * 4), "allocate pinned C");
            }
            if (ok) parallel_spans(m, std::max(1, host_cpus() / o.gpus), [&](size_t lo, size_t hi) {
                b200va_host_fill_ctr_f32(hA + lo, hi - lo, o.seed, b + lo);
                b200va_host_fill_ctr_f32(hB + lo, hi - lo, o.seed + 1, b + lo);
            });
            VA(b200va_stager_create(&stager, rank, 0, 0), "create stager");
        } else {
            CK(cudaMalloc(&dA, m ? m * 4 : 4), "allocate device vector A");
            CK(cudaMalloc(&dB, m ? m * 4 : 4), "allocate device vector B");
            CK(cudaMalloc(&dC, m ? m * 4 : 4), "allocate device vector C");
            VA(b200va_fill_ctr_f32(dA, m, o.seed, b, st), "generate A");   // global index => sharding invisible
            VA(b200va_fill_ctr_f32(dB, m, o.seed + 1, b, st), "generate B");
            // warm-up
            VA(b200va_loop_create(&loop, dA, dB, dC, m, o.variant, o.graph), "capture launch loop");
            VA(b200va_loop_run(loop, std::max(3, o.graph), st), "warm up");
            CK(cudaStreamSynchronize(st), "warm up");
        }
    }

    double last_ms_per_pass = 0.0;
    auto run_block = [&](int count) {   // one block of `count` passes, event-timed
        const double before = r.gpu_ms;
        if (staged) {
            for (int i = 0; i < count && ok; ++i) {
                const auto w0 = clk::now();
                VA(b200va_stager_add_f32(stager, hA, hB, hC, m, o.variant, o.stage_mode), "staged add");
                float ms = 0; if (ok) b200va_stager_last_ms(stager, &ms);
                if (r.launches + i == 0) {
                    r.first_pass_wall_ms = secs_since(w0) * 1e3;   // includes one-off page-locking
                    if (ok) b200va_stager_last_mode(stager, &r.first_stage_mode);
                }
                r.gpu_ms += ms;
            }
            if (ok) b200va_stager_last_mode(stager, &r.stage_mode);
        } else {
            CK(cudaEventRecord(e0, st), "record event");
            VA(b200va_loop_run(loop, count, st), "launch vectorAdd kernel");
            CK(cudaEventRecord(e1, st), "record event");
            CK(cudaEventSynchronize(e1), "synchronize");
            float ms = 0; if (ok) CK(cudaEventElapsedTime(&ms, e0, e1), "read event");
            r.gpu_ms += ms;
        }
        r.launches += count;
        if (count > 0) last_ms_per_pass = (r.gpu_ms - before) / count;
    };

    bar.wait();
    const auto t0 = clk::now();
    if (o.duration <= 0) {
        if (ok) run_block(o.iters);
    } else {
        const double period = o.period_ms * 1e-3;
        double next_sample = 0.0;
        while (ok && secs_since(t0) < o.duration) {
            const auto p0 = clk::now();
            if (o.target_util > 0) {     // busy for target% of the period, then idle
                // busy budget of this period, spent in blocks of at most --iters passes; the block is
                // shrunk to what still fits so that small targets (a few %) are not overshot
                const double budget = period * o.target_util / 100.0;
                do {
                    int count = o.iters;
                    if (last_ms_per_pass > 0) {
                        const double fit = (budget - secs_since(p0)) * 1e3 / last_ms_per_pass;
                        count = static_cast<int>(std::max(1.0, std::min(static_cast<double>(o.iters), fit)));
                    }
                    run_block(count);
                } while (ok && secs_since(p0) < budget - 0.5e-3 * last_ms_per_pass);
                const double rest = period - secs_since(p0);
                if (rest > 0) std::this_thread::sleep_for(std::chrono::duration<double>(rest));
            } else {
                run_block(o.iters);
            }
            if (nvml && secs_since(t0) >= next_sample) {
                r.util_samples.push_back(nvml->gpu_util(static_cast<size_t>(rank)));
                if (!o.metrics_file.empty() && rank == 0) nvml->write_metrics(o.metrics_file, 0, r.util_samples.back());
                next_sample += 0.5;
            }
        }
    }
    r.wall_s = secs_since(t0);
    bar.wait();

    if (ok && o.verify) {
        if (staged) {
            std::atomic<size_t> first{~size_t{0}};
            parallel_spans(m, std::max(1, host_cpus() / o.gpus), [&](size_t lo, size_t hi) {
                size_t bad = 0;
                if (b200va_host_verify_f32(hA + lo, hB + lo, hC + lo, hi - lo, &bad) != B200VA_OK) {
                    size_t cur = first.load();
                    while (lo + bad < cur && !first.compare_exchange_weak(cur, lo + bad)) {}
                }
            });
            if (first.load() != ~size_t{0}) { r.mismatches = 1; r.first_bad = b + first.load(); }
        } else {
            uint64_t h[4] = {0, 0, 0, 0};
            VA(b200va_verify_f32(dA, dB, dC, m, dRes, st), "verify on device");
            VA(b200va_digest_f32(dC, m, dRes + 2, st), "digest on device");
            CK(cudaMemcpyAsync(h, dRes, sizeof h, cudaMemcpyDeviceToHost, st), "copy verdict");
            CK(cudaStreamSynchronize(st), "synchronize");
            r.mismatches = h[0]; r.first_bad = h[0] ? b + h[1] : ~0ull; r.digest[0] = h[2]; r.digest[1] = h[3];
        }
    }
    if (st) cudaStreamSynchronize(st);
    if (loop) b200va_loop_destroy(loop);
    if (stager) b200va_stager_destroy(stager);    // unregisters the malloc'd arrays before they are freed
    if (staged && o.pageable) { std::free(hA); std::free(hB); std::free(hC); }
    else { b200va_host_free(hA); b200va_host_free(hB); b200va_host_free(hC); }
    cudaFree(dA); cudaFree(dB); cudaFree(dC); cudaFree(dRes);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    if (st) cudaStreamDestroy(st);
}

int run_sharded(const Options& o)
{
    int ndev = 0;
    ck(cudaGetDeviceCount(&ndev), "count CUDA devices");
    if (ndev < o.gpus) {
        std::fprintf(stderr, "Failed to find %d CUDA devices (found %d)!\n", o.gpus, ndev);
        return EXIT_FAILURE;
    }
    b200va_devinfo_t di;
    for (int d = 0; d < o.gpus; ++d) va(b200va_query(d, &di), "find an H100-class CUDA device");

    Nvml nvml;
    bool have_nvml = false;
    if (o.nvml) {
        std::vector<int> devs;
        for (int d = 0; d < o.gpus; ++d) devs.push_back(d);
        have_nvml = nvml.open(devs);
        if (!have_nvml) std::fprintf(stderr, "warning: NVML unavailable, utilisation not sampled\n");
    }

    CpuBaseline cpu;
    if (o.cpu_baseline) cpu = run_cpu_baseline(std::min(o.n, size_t{1} << 28), o.cpu_threads);

    Barrier bar(o.gpus);
    std::vector<ShardResult> res(static_cast<size_t>(o.gpus));
    std::vector<std::thread> th;
    for (int g = 0; g < o.gpus; ++g)
        th.emplace_back(shard_worker, std::cref(o), g, std::ref(bar), std::ref(res[static_cast<size_t>(g)]),
                        have_nvml ? &nvml : nullptr);
    for (auto& t : th) t.join();

    double max_ms = 0, max_wall = 0;
    long long launches = 0;
    uint64_t mism = 0, first_bad = ~0ull, dig[2] = {0, 0};
    for (auto& r : res) {
        if (!r.error.empty()) {
            std::fprintf(stderr, "Failed to %s!\n", r.error.c_str());
            return EXIT_FAILURE;
        }
        max_ms = std::max(max_ms, r.gpu_ms);
        max_wall = std::max(max_wall, r.wall_s);
        launches = std::max(launches, r.launches);
        mism += r.mismatches;
        first_bad = std::min(first_bad, r.first_bad);
        dig[0] += r.digest[0];
        dig[1] ^= r.digest[1];
    }
    const double elems = static_cast<double>(o.n) * static_cast<double>(launches);
    const double eps = max_ms > 0 ? elems / (max_ms * 1e-3) : 0.0;
    const double gbps = eps * 12.0 / 1e9;
    b200va_tune_t tune;
    b200va_resolve(o.variant, (o.n + static_cast<size_t>(o.gpus) - 1) / static_cast<size_t>(o.gpus), &tune);

    std::string js;
    char buf[1024];
    std::snprintf(buf, sizeof buf,
                  "{\"metric\": \"fp32 elements/sec\", \"mode\": \"%s\", \"n\": %zu, \"gpus\": %d, \"kernel\": \"%s\", "
                  "\"iters_per_block\": %d, \"launches_per_gpu\": %lld, \"graph_batch\": %d, \"gpu_ms_max\": %.4f, "
                  "\"ms_per_pass\": %.5f, \"elements_per_s\": %.5e, \"algorithmic_GBps\": %.1f, "
                  "\"roofline_frac_of_3p35TBps_per_gpu\": %.4f, \"wall_s\": %.4f, \"gpu_busy_frac\": %.4f, "
                  "\"mismatches\": %" PRIu64 ", \"digest_sum\": \"%016" PRIx64 "\", \"digest_xor\": \"%08" PRIx64 "\"",
                  o.mode.c_str(), o.n, o.gpus, variant_name(tune.kind), o.iters, launches, o.graph, max_ms,
                  launches ? max_ms / static_cast<double>(launches) : 0.0, eps, gbps, gbps / (3350.0 * o.gpus), max_wall,
                  max_wall > 0 ? max_ms * 1e-3 / max_wall : 0.0, mism, dig[0], dig[1]);
    js = buf;
    if (o.mode == "staged") {
        std::snprintf(buf, sizeof buf, ", \"host_mem\": \"%s\", \"first_stage_mode\": %d, \"stage_mode\": %d, \"first_pass_wall_ms\": %.3f",
                      o.pageable ? "pageable (malloc)" : "pinned (b200va_host_alloc)", res[0].first_stage_mode, res[0].stage_mode,
                      res[0].first_pass_wall_ms);
        js += buf;
    }
    if (have_nvml) {
        double sum = 0; int cnt = 0, mx = 0;
        for (auto& r : res) for (int u : r.util_samples) if (u >= 0) { sum += u; ++cnt; mx = std::max(mx, u); }
        const double mean = cnt ? sum / cnt : 0.0;
        std::snprintf(buf, sizeof buf, ", \"nvml_util_mean\": %.1f, \"nvml_util_max\": %d, \"nvml_samples\": %d, "
                      "\"hpa_threshold\": %.1f, \"hpa_tolerance\": 0.1, \"hpa_ratio\": %.4f, \"hpa_would_scale\": %s, "
                      "\"nvml_sample_period_s\": 0.5, \"nvml_trace\": [",
                      mean, mx, cnt, o.hpa_threshold, o.hpa_threshold > 0 ? mean / o.hpa_threshold : 0.0,
                      // the controller acts only outside its 10 % tolerance band (hpa_replay.hpa_desired_replicas)
                      mean > o.hpa_threshold * 1.1 ? "true" : "false");
        js += buf;
        for (size_t g = 0; g < res.size(); ++g) {          // one utilisation trace per GPU (0.5 s apart)
            js += g ? ", [" : "[";
            for (size_t i = 0; i < res[g].util_samples.size(); ++i) {
                std::snprintf(buf, sizeof buf, "%s%d", i ? ", " : "", res[g].util_samples[i]);
                js += buf;
            }
            js += "]";
        }
        js += "]";
    }
    if (o.cpu_baseline) {
        std::snprintf(buf, sizeof buf, ", \"cpu_baseline\": {\"n\": %zu, \"threads\": %d, \"ms_median\": %.3f, "
                      "\"elements_per_s\": %.4e, \"algorithmic_GBps\": %.2f, \"stores\": \"regular (write-allocate)\"}, "
                      "\"gpu_over_cpu\": %.1f", cpu.n, cpu.threads, cpu.ms_median, cpu.elems_per_s, cpu.gbps,
                      cpu.elems_per_s > 0 ? eps / cpu.elems_per_s : 0.0);
        js += buf;
    }
    js += "}";
    std::printf("%s\n", js.c_str());
    if (!o.json_path.empty()) {
        if (FILE* f = std::fopen(o.json_path.c_str(), "w")) { std::fprintf(f, "%s\n", js.c_str()); std::fclose(f); }
        else { std::fprintf(stderr, "Failed to write %s!\n", o.json_path.c_str()); return EXIT_FAILURE; }
    }
    if (o.verify && mism) {
        std::fprintf(stderr, "Result verification failed at element %" PRIu64 "!\n", first_bad);
        return EXIT_FAILURE;
    }
    return EXIT_SUCCESS;
}

}  // namespace

int main(int argc, char** argv)
{
    const Options o = parse(argc, argv);
    if (o.mode == "sample") return run_sample(o);
    return run_sharded(o);
}
