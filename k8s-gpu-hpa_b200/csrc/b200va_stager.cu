// b200va_stager.cu -- the host-buffer path of libb200va.so: the copy pool, NUMA-local pinned
// allocation, register-once and the chunk pipelines that feed the f32 add from host arrays.
// Host code only: the adds go through the same launch as b200va_add_f32 (b200va_add.cu).
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <cctype>
#include <condition_variable>
#include <thread>
#include <vector>

#include "b200va_internal.h"

using namespace b200va;

// ------------------------------------------------------------------ host-buffer path
// Fork-join pool for the pageable path: T persistent workers, each copies one slice.
// Construction may throw (std::system_error from std::thread under a pids limit, bad_alloc):
// make_copy_pool() catches and degrades, nothing propagates through the C ABI.
class CopyPool {
public:
    explicit CopyPool(int threads) : n_(threads < 1 ? 1 : threads)
    {
        th_.reserve(static_cast<size_t>(n_));
        try {
            for (int i = 1; i < n_; ++i) th_.emplace_back([this, i] { worker(i); });
        } catch (...) {
            n_ = static_cast<int>(th_.size()) + 1;          // run with the workers that did start
        }
    }
    ~CopyPool()
    {
        { std::lock_guard<std::mutex> lk(m_); stop_ = true; ++gen_; }
        cv_.notify_all();
        for (auto& t : th_) t.join();
    }
    int size() const { return n_; }
    // dst[0..bytes) = src[0..bytes), split in 64-byte-aligned slices over the pool (caller = slice 0)
    void copy(void* dst, const void* src, size_t bytes)
    {
        if (bytes < (size_t{1} << 20) || n_ == 1) { std::memcpy(dst, src, bytes); return; }
        {
            std::lock_guard<std::mutex> lk(m_);
            dst_ = static_cast<unsigned char*>(dst); src_ = static_cast<const unsigned char*>(src); bytes_ = bytes;
            pending_ = n_ - 1;
            ++gen_;
        }
        cv_.notify_all();
        slice(0);
        std::unique_lock<std::mutex> lk(m_);
        done_.wait(lk, [this] { return pending_ == 0; });
    }

private:
    void slice(int i)
    {
        size_t per = (bytes_ + static_cast<size_t>(n_) - 1) / static_cast<size_t>(n_);
        per = (per + 63) & ~size_t{63};
        const size_t lo = std::min(bytes_, per * static_cast<size_t>(i)), hi = std::min(bytes_, lo + per);
        if (hi > lo) std::memcpy(dst_ + lo, src_ + lo, hi - lo);
    }
    void worker(int i)
    {
        unsigned long seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lk(m_);
                cv_.wait(lk, [&] { return gen_ != seen; });
                seen = gen_;
                if (stop_) return;
            }
            if (i < n_) slice(i);
            std::lock_guard<std::mutex> lk(m_);
            if (--pending_ == 0) done_.notify_one();
        }
    }
    int n_;
    std::vector<std::thread> th_;
    std::mutex m_;
    std::condition_variable cv_, done_;
    unsigned long gen_ = 0;
    int pending_ = 0;
    bool stop_ = false;
    unsigned char* dst_ = nullptr;
    const unsigned char* src_ = nullptr;
    size_t bytes_ = 0;
};

// Copy threads: the CPUs this process may use (affinity mask, cgroup v2 bandwidth quota), at
// most 16; B200VA_COPY_THREADS overrides (clamped to 1..64).  Never throws: returns nullptr
// only if even a single-threaded pool cannot be allocated.
static CopyPool* make_copy_pool()
{
    unsigned hw = std::thread::hardware_concurrency();
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof set, &set) == 0 && CPU_COUNT(&set) > 0) hw = static_cast<unsigned>(CPU_COUNT(&set));
    if (FILE* f = std::fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char q[64];
        double period = 0;
        if (std::fscanf(f, "%63s %lf", q, &period) == 2 && std::strcmp(q, "max") != 0 && period > 0)
            hw = std::min(hw, static_cast<unsigned>(std::max(1.0, std::atof(q) / period)));
        std::fclose(f);
    }
    unsigned want = std::max(1u, std::min(16u, hw));
    if (const char* e = std::getenv("B200VA_COPY_THREADS")) want = static_cast<unsigned>(std::min(64, std::max(1, std::atoi(e))));
    for (; want >= 1; want /= 2) {
        try {
            return new CopyPool(static_cast<int>(want));
        } catch (...) {
            // bad_alloc / system_error while building the pool: retry smaller
        }
        if (want == 1) break;
    }
    return nullptr;
}

struct HostRange { uintptr_t lo, hi; };     // [lo, hi) page-locked by this stager (mode 4)

struct b200va_stager {
    int device = 0;
    size_t chunk = 0;
    int depth = 0;
    float* d_buf = nullptr;            // depth * 3 * chunk floats
    cudaStream_t main = nullptr;
    cudaStream_t* slot = nullptr;
    cudaEvent_t* slot_done = nullptr;
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
    // "lanes" pipeline (mode 2): one stream per direction + one for the kernel, events per slot
    cudaStream_t lane_h2d = nullptr, lane_k = nullptr, lane_d2h = nullptr;
    cudaEvent_t *ev_in = nullptr, *ev_sum = nullptr, *ev_out = nullptr;
    // pageable path (mode 3): pinned bounce chunks (depth * 3 * bounce_chunk floats) + copy threads, made on first use
    float* bounce = nullptr;
    size_t bounce_chunk = 0;
    CopyPool* pool = nullptr;
    // register-once path (mode 4): host ranges this stager page-locked
    std::vector<HostRange>* regs = nullptr;
    float last_ms = 0.f;
    int last_mode = -1;
};

// NUMA node a CUDA device hangs off (sysfs), or -1.  B200VA_NUMA_NODE overrides.
static int device_numa_node_of(int dev)
{
    if (const char* e = std::getenv("B200VA_NUMA_NODE")) return std::atoi(e);
    char bus[32] = {0}, path[128];
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, dev) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char* c = bus; *c; ++c) *c = static_cast<char>(std::tolower(*c));
    std::snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    int node = -1;
    if (FILE* f = std::fopen(path, "r")) {
        if (std::fscanf(f, "%d", &node) != 1) node = -1;
        std::fclose(f);
    }
    return node;
}

static int device_numa_node()
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return -1; }
    return device_numa_node_of(dev);
}

// Parses a sysfs cpulist ("0-31,64-95") into a cpu_set_t restricted to `allowed`.
static bool node_cpuset(int node, const cpu_set_t& allowed, cpu_set_t* out)
{
    char path[96], buf[4096];
    std::snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    FILE* f = std::fopen(path, "r");
    if (!f) return false;
    const bool ok = std::fgets(buf, sizeof buf, f) != nullptr;
    std::fclose(f);
    if (!ok) return false;
    CPU_ZERO(out);
    int count = 0;
    for (char* p = buf; *p && *p != '\n';) {
        char* end = nullptr;
        long lo = std::strtol(p, &end, 10), hi = lo;
        if (end == p) break;
        if (*end == '-') hi = std::strtol(end + 1, &end, 10);
        for (long c = lo; c <= hi && c < CPU_SETSIZE; ++c)
            if (CPU_ISSET(c, &allowed)) { CPU_SET(c, out); ++count; }
        p = (*end == ',') ? end + 1 : end;
    }
    return count > 0;
}

// Pinned, mapped host memory whose pages sit on the NUMA node local to the current GPU:
// the calling thread is moved onto that node's CPUs (and its memory policy set to prefer
// the node) for the duration of the allocation, so the first touch inside cudaHostAlloc
// lands there; a PCIe DMA then never crosses the inter-socket link.  Affinity and memory
// policy of the caller (e.g. numactl --interleave) are saved and put back.
int b200va_host_alloc_ex(void** out, size_t bytes, int write_combined)
{
    if (!out) return B200VA_ERR_INVALID;
    const int node = device_numa_node();
    cpu_set_t old_set, node_set;
    bool moved = false, policy = false;
    int old_mode = 0;
    unsigned long old_mask[16] = {0};                       // 1024 nodes
    constexpr unsigned long kMaxNode = sizeof old_mask * 8;
    if (node >= 0 && sched_getaffinity(0, sizeof old_set, &old_set) == 0 && node_cpuset(node, old_set, &node_set)) {
        moved = sched_setaffinity(0, sizeof node_set, &node_set) == 0;
        if (node < 64 && syscall(SYS_get_mempolicy, &old_mode, old_mask, kMaxNode, nullptr, 0ul) == 0) {
            unsigned long mask = 1ul << node;
            policy = syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, &mask, 65ul) == 0;
        }
    }
    unsigned flags = cudaHostAllocPortable | cudaHostAllocMapped;
    if (write_combined) flags |= cudaHostAllocWriteCombined;   // H2D sources only: CPU reads of WC memory crawl
    const cudaError_t e = cudaHostAlloc(out, bytes ? bytes : 1, flags);
    if (policy) {
        bool any = false;
        for (unsigned long w : old_mask) any = any || w != 0;
        if (syscall(SYS_set_mempolicy, old_mode, any ? old_mask : nullptr, any ? kMaxNode : 0ul) != 0)
            syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0ul);
    }
    if (moved) sched_setaffinity(0, sizeof old_set, &old_set);
    CU_TRY(e);
    return B200VA_OK;
}

int b200va_host_alloc(void** out, size_t bytes) { return b200va_host_alloc_ex(out, bytes, 0); }

// NUMA node the current CUDA device is attached to (sysfs), or -1.
int b200va_device_numa_node(void) { return device_numa_node(); }
int b200va_device_numa_node_of(int device) { return device_numa_node_of(device); }

// NUMA node holding the page at `p` (get_mempolicy(MPOL_F_NODE | MPOL_F_ADDR)), or -1.
int b200va_host_node_of(const void* p)
{
    int node = -1;
    if (!p) return -1;
    if (syscall(SYS_get_mempolicy, &node, nullptr, 0ul, const_cast<void*>(p), 3ul /* F_NODE|F_ADDR */) != 0) return -1;
    return node;
}

int b200va_host_free(void* p)
{
    if (!p) return B200VA_OK;
    CU_TRY(cudaFreeHost(p));
    return B200VA_OK;
}

static void stager_release_host(b200va_stager* s)
{
    if (!s->regs) return;
    for (const HostRange& r : *s->regs)
        if (cudaHostUnregister(reinterpret_cast<void*>(r.lo)) != cudaSuccess) cudaGetLastError();
    s->regs->clear();
}

int b200va_stager_release_host(b200va_stager_t* s)
{
    if (!s) return B200VA_ERR_INVALID;
    DeviceGuard g(s->device);
    stager_release_host(s);
    return B200VA_OK;
}

int b200va_stager_destroy(b200va_stager_t* s)
{
    if (!s) return B200VA_OK;
    DeviceGuard g(s->device);
    stager_release_host(s);
    delete s->regs;
    if (s->slot) {
        for (int i = 0; i < s->depth; ++i) {
            if (s->slot[i]) cudaStreamDestroy(s->slot[i]);
            if (s->slot_done && s->slot_done[i]) cudaEventDestroy(s->slot_done[i]);
        }
    }
    for (cudaStream_t st : {s->lane_h2d, s->lane_k, s->lane_d2h})
        if (st) cudaStreamDestroy(st);
    for (cudaEvent_t* arr : {s->ev_in, s->ev_sum, s->ev_out}) {
        if (!arr) continue;
        for (int i = 0; i < s->depth; ++i)
            if (arr[i]) cudaEventDestroy(arr[i]);
        delete[] arr;
    }
    if (s->main) cudaStreamDestroy(s->main);
    if (s->ev_start) cudaEventDestroy(s->ev_start);
    if (s->ev_stop) cudaEventDestroy(s->ev_stop);
    if (s->d_buf) cudaFree(s->d_buf);
    if (s->bounce) cudaFreeHost(s->bounce);
    delete s->pool;
    delete[] s->slot;
    delete[] s->slot_done;
    delete s;
    return B200VA_OK;
}

int b200va_stager_create(b200va_stager_t** out, int device, size_t chunk_elems, int depth)
{
    if (!out) return B200VA_ERR_INVALID;
    *out = nullptr;
    if (chunk_elems == 0) chunk_elems = size_t{1} << 25;   // 128 MiB per array per slot (the lanes pipeline tapers the tail)
    if (depth == 0) depth = 3;
    if (depth < 1 || depth > 16) return B200VA_ERR_INVALID;
    chunk_elems = (chunk_elems + 63) & ~size_t{63};        // slots stay 256-B aligned
    RC_TRY(dev_info(device, nullptr));
    DeviceGuard guard(device);
    CU_TRY(guard.err);
    b200va_stager* s = new (std::nothrow) b200va_stager;
    if (!s) return B200VA_ERR_NOMEM;
    s->device = device;
    s->chunk = chunk_elems;
    s->depth = depth;
    s->slot = new (std::nothrow) cudaStream_t[depth]();
    s->slot_done = new (std::nothrow) cudaEvent_t[depth]();
    s->regs = new (std::nothrow) std::vector<HostRange>();
    if (!s->slot || !s->slot_done || !s->regs) { b200va_stager_destroy(s); return B200VA_ERR_NOMEM; }
    cudaError_t e = cudaMalloc(&s->d_buf, static_cast<size_t>(depth) * 3 * chunk_elems * sizeof(float));
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->main, cudaStreamNonBlocking);
    for (int i = 0; i < depth && e == cudaSuccess; ++i) {
        e = cudaStreamCreateWithFlags(&s->slot[i], cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->slot_done[i], cudaEventDisableTiming);
    }
    if (e == cudaSuccess) e = cudaEventCreate(&s->ev_start);
    if (e == cudaSuccess) e = cudaEventCreate(&s->ev_stop);
    s->ev_in = new (std::nothrow) cudaEvent_t[depth]();
    s->ev_sum = new (std::nothrow) cudaEvent_t[depth]();
    s->ev_out = new (std::nothrow) cudaEvent_t[depth]();
    if (!s->ev_in || !s->ev_sum || !s->ev_out) { b200va_stager_destroy(s); return B200VA_ERR_NOMEM; }
    for (cudaStream_t* st : {&s->lane_h2d, &s->lane_k, &s->lane_d2h})
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(st, cudaStreamNonBlocking);
    for (int i = 0; i < depth && e == cudaSuccess; ++i) {
        e = cudaEventCreateWithFlags(&s->ev_in[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->ev_sum[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->ev_out[i], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) { b200va_stager_destroy(s); return cuda_err(e); }
    *out = s;
    return B200VA_OK;
}

// ---- the pipelines (device already current; a non-OK return leaves work in flight: the caller drains)
static int stage_zero_copy(b200va_stager* s, const float* hA, const float* hB, float* hC, size_t n, int variant)
{
    // the kernel streams A and B from pinned host memory over PCIe and writes C back the same
    // way -- both link directions busy, no staging latency.
    const float *dA = nullptr, *dB = nullptr;
    float* dC = nullptr;
    if (n) {
        CU_TRY(cudaHostGetDevicePointer(reinterpret_cast<void**>(const_cast<float**>(&dA)), const_cast<float*>(hA), 0));
        CU_TRY(cudaHostGetDevicePointer(reinterpret_cast<void**>(const_cast<float**>(&dB)), const_cast<float*>(hB), 0));
        CU_TRY(cudaHostGetDevicePointer(reinterpret_cast<void**>(&dC), hC, 0));
    }
    b200va_tune_t t;
    default_tune(variant == B200VA_K_AUTO ? B200VA_K1_VEC128 : variant, n, &t);
    return launch(dA, dB, dC, n, t, s->main, pdl_enabled());
}

static int stage_slots(b200va_stager* s, const float* hA, const float* hB, float* hC, size_t n, int variant)
{
    const size_t nchunks = (n + s->chunk - 1) / s->chunk;
    for (int i = 0; i < s->depth; ++i) CU_TRY(cudaStreamWaitEvent(s->slot[i], s->ev_start, 0));
    b200va_tune_t t;
    for (size_t k = 0; k < nchunks; ++k) {
        const int i = static_cast<int>(k % static_cast<size_t>(s->depth));
        const size_t off = k * s->chunk;
        const size_t m = (n - off < s->chunk) ? n - off : s->chunk;
        float* dA = s->d_buf + static_cast<size_t>(i) * 3 * s->chunk;
        float* dB = dA + s->chunk;
        float* dC = dB + s->chunk;
        CU_TRY(cudaMemcpyAsync(dA, hA + off, m * sizeof(float), cudaMemcpyHostToDevice, s->slot[i]));
        CU_TRY(cudaMemcpyAsync(dB, hB + off, m * sizeof(float), cudaMemcpyHostToDevice, s->slot[i]));
        default_tune(variant, m, &t, B200VA_F_COLD);      // a chunk fresh off the copy engine is never in L2
        RC_TRY(launch(dA, dB, dC, m, t, s->slot[i], pdl_enabled()));
        CU_TRY(cudaMemcpyAsync(hC + off, dC, m * sizeof(float), cudaMemcpyDeviceToHost, s->slot[i]));
    }
    for (int i = 0; i < s->depth; ++i) {
        CU_TRY(cudaEventRecord(s->slot_done[i], s->slot[i]));
        CU_TRY(cudaStreamWaitEvent(s->main, s->slot_done[i], 0));
    }
    return B200VA_OK;
}

// Fault injection for the error-path test (tests/test_gpu_host_path.py): with
// B200VA_TEST_FAIL_CHUNK=k in the environment the lanes pipeline fails ONCE per process, right
// after it has queued chunk k's H2D copies -- i.e. with DMA in flight on the caller's arrays.
static bool inject_fault_at_chunk(size_t k)
{
    static const long at = [] { const char* e = std::getenv("B200VA_TEST_FAIL_CHUNK"); return e ? std::atol(e) : -1L; }();
    static std::atomic<bool> fired{false};
    return at >= 0 && static_cast<long>(k) == at && !fired.exchange(true);
}

static int stage_lanes(b200va_stager* s, const float* hA, const float* hB, float* hC, size_t n, int variant)
{
    // lanes: every H2D copy queues on one stream, every add on a second, every D2H on a
    // third; slot reuse and data flow are event edges.  The H2D queue -- the bottleneck
    // direction -- never waits behind a kernel or a D2H of another chunk.
    for (cudaStream_t st : {s->lane_h2d, s->lane_k, s->lane_d2h}) CU_TRY(cudaStreamWaitEvent(st, s->ev_start, 0));
    b200va_tune_t t;
    // Full-size chunks, then a tapered tail (1/2, 1/4, ... down to ~1 Mi elements): what is left
    // after the last H2D byte has arrived is one small add and one small D2H, not a full chunk.
    const size_t taper_min = size_t{1} << 20;
    size_t off = 0;
    for (size_t k = 0; off < n; ++k) {
        const size_t left = n - off;
        size_t m = s->chunk;
        if (left <= s->chunk && s->depth > 1) {
            m = left / 2;
            m = (m + 63) & ~size_t{63};                      // chunk starts stay 256-byte aligned
            if (m < taper_min || m >= left) m = left;
        }
        if (m > left) m = left;
        const int i = static_cast<int>(k % static_cast<size_t>(s->depth));
        float* dA = s->d_buf + static_cast<size_t>(i) * 3 * s->chunk;
        float* dB = dA + s->chunk;
        float* dC = dB + s->chunk;
        if (k >= static_cast<size_t>(s->depth)) CU_TRY(cudaStreamWaitEvent(s->lane_h2d, s->ev_out[i], 0));  // slot drained
        CU_TRY(cudaMemcpyAsync(dA, hA + off, m * sizeof(float), cudaMemcpyHostToDevice, s->lane_h2d));
        CU_TRY(cudaMemcpyAsync(dB, hB + off, m * sizeof(float), cudaMemcpyHostToDevice, s->lane_h2d));
        CU_TRY(cudaEventRecord(s->ev_in[i], s->lane_h2d));
        if (inject_fault_at_chunk(k)) return B200VA_ERR_INVALID;   // test hook: fail with copies in flight
        CU_TRY(cudaStreamWaitEvent(s->lane_k, s->ev_in[i], 0));
        default_tune(variant, m, &t, B200VA_F_COLD);      // a chunk fresh off the copy engine is never in L2
        RC_TRY(launch(dA, dB, dC, m, t, s->lane_k, pdl_enabled()));
        CU_TRY(cudaEventRecord(s->ev_sum[i], s->lane_k));
        CU_TRY(cudaStreamWaitEvent(s->lane_d2h, s->ev_sum[i], 0));
        CU_TRY(cudaMemcpyAsync(hC + off, dC, m * sizeof(float), cudaMemcpyDeviceToHost, s->lane_d2h));
        CU_TRY(cudaEventRecord(s->ev_out[i], s->lane_d2h));
        off += m;
    }
    CU_TRY(cudaEventRecord(s->slot_done[0], s->lane_d2h));   // the D2H lane finishes last
    CU_TRY(cudaStreamWaitEvent(s->main, s->slot_done[0], 0));
    return B200VA_OK;
}

static int stage_bounce(b200va_stager* s, const float* hA, const float* hB, float* hC, size_t n, int variant)
{
    // Pageable host arrays (plain malloc, what one ./vectorAdd process has): a cudaMemcpy from
    // pageable memory is staged by the driver on one thread at ~10 GB/s.  Here a pool of host
    // threads copies chunk k+1 into pinned bounce buffers and chunk k-2 out of them while the
    // copy engines and the add work on the chunks in between (lanes as in mode 2).
    const size_t bc = std::min(s->chunk, size_t{1} << 23);          // 32 MiB bounce chunks
    if (!s->pool) {
        s->pool = make_copy_pool();
        if (!s->pool) return B200VA_ERR_NOMEM;
    }
    if (!s->bounce || s->bounce_chunk != bc) {
        if (s->bounce) { cudaFreeHost(s->bounce); s->bounce = nullptr; }
        void* p = nullptr;
        RC_TRY(b200va_host_alloc(&p, static_cast<size_t>(s->depth) * 3 * bc * sizeof(float)));
        s->bounce = static_cast<float*>(p);
        s->bounce_chunk = bc;
    }
    for (cudaStream_t st : {s->lane_h2d, s->lane_k, s->lane_d2h}) CU_TRY(cudaStreamWaitEvent(st, s->ev_start, 0));
    const size_t nchunks = (n + bc - 1) / bc;
    const size_t depth = static_cast<size_t>(s->depth);
    b200va_tune_t t;
    auto span = [&](size_t k, size_t* off, size_t* m) { *off = k * bc; *m = std::min(bc, n - *off); };
    for (size_t k = 0; k < nchunks + depth - 1 || k < nchunks; ++k) {
        if (k < nchunks) {
            size_t off, m;
            span(k, &off, &m);
            const size_t i = k % depth;
            float* pA = s->bounce + i * 3 * bc;
            float* dA = s->d_buf + i * 3 * s->chunk;
            // slot i was drained (copied out) at iteration k-1 below, or never used
            s->pool->copy(pA, hA + off, m * sizeof(float));
            s->pool->copy(pA + bc, hB + off, m * sizeof(float));
            CU_TRY(cudaMemcpyAsync(dA, pA, m * sizeof(float), cudaMemcpyHostToDevice, s->lane_h2d));
            CU_TRY(cudaMemcpyAsync(dA + s->chunk, pA + bc, m * sizeof(float), cudaMemcpyHostToDevice, s->lane_h2d));
            CU_TRY(cudaEventRecord(s->ev_in[i], s->lane_h2d));
            CU_TRY(cudaStreamWaitEvent(s->lane_k, s->ev_in[i], 0));
            default_tune(variant, m, &t, B200VA_F_COLD);
            RC_TRY(launch(dA, dA + s->chunk, dA + 2 * s->chunk, m, t, s->lane_k, pdl_enabled()));
            CU_TRY(cudaEventRecord(s->ev_sum[i], s->lane_k));
            CU_TRY(cudaStreamWaitEvent(s->lane_d2h, s->ev_sum[i], 0));
            CU_TRY(cudaMemcpyAsync(pA + 2 * bc, dA + 2 * s->chunk, m * sizeof(float), cudaMemcpyDeviceToHost, s->lane_d2h));
            CU_TRY(cudaEventRecord(s->ev_out[i], s->lane_d2h));
        }
        if (k + 1 >= depth) {                                       // retire chunk j = k - (depth - 1)
            const size_t j = k + 1 - depth;
            if (j < nchunks) {
                size_t off, m;
                span(j, &off, &m);
                const size_t i = j % depth;
                CU_TRY(cudaEventSynchronize(s->ev_out[i]));
                s->pool->copy(hC + off, s->bounce + i * 3 * bc + 2 * bc, m * sizeof(float));
            }
        }
    }
    CU_TRY(cudaEventRecord(s->slot_done[0], s->lane_d2h));
    CU_TRY(cudaStreamWaitEvent(s->main, s->slot_done[0], 0));
    return B200VA_OK;
}

static bool host_is_pinned(const void* p)
{
    cudaPointerAttributes at{};
    const bool ok = cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type != cudaMemoryTypeUnregistered;
    if (!ok) cudaGetLastError();
    return ok;
}

// Page-locks [p, p+bytes) in place unless the runtime already knows it (cudaHostAlloc'd,
// registered by the caller, or by this stager earlier).  Returns false if the range cannot be
// registered -- the caller then falls back to the bounce path.
static bool ensure_registered(b200va_stager* s, const void* p, size_t bytes)
{
    if (bytes == 0) return true;
    const uintptr_t lo = reinterpret_cast<uintptr_t>(p), hi = lo + bytes;
    for (const HostRange& r : *s->regs)
        if (r.lo <= lo && hi <= r.hi) return true;                  // cached
    if (host_is_pinned(p) && host_is_pinned(reinterpret_cast<const void*>(hi - 1))) return true;
    // a cached range that overlaps without containing the new one (the caller's buffer moved or grew): drop it
    for (size_t i = 0; i < s->regs->size();) {
        const HostRange r = (*s->regs)[i];
        if (r.lo < hi && lo < r.hi) {
            if (cudaHostUnregister(reinterpret_cast<void*>(r.lo)) != cudaSuccess) cudaGetLastError();
            s->regs->erase(s->regs->begin() + static_cast<long>(i));
        } else {
            ++i;
        }
    }
    const cudaError_t e = cudaHostRegister(const_cast<void*>(p), bytes, cudaHostRegisterPortable);
    if (e != cudaSuccess) { cudaGetLastError(); return false; }
    try {
        s->regs->push_back(HostRange{lo, hi});
    } catch (...) {
        cudaHostUnregister(const_cast<void*>(p));
        return false;
    }
    return true;
}

static void stager_drain(b200va_stager* s)
{
    // after a failure in the middle of a pipeline: nothing may still be reading or writing the
    // caller's arrays (or the bounce ring) when the error code is returned
    for (int i = 0; i < s->depth; ++i)
        if (s->slot && s->slot[i]) cudaStreamSynchronize(s->slot[i]);
    for (cudaStream_t st : {s->lane_h2d, s->lane_k, s->lane_d2h, s->main})
        if (st) cudaStreamSynchronize(st);
    cudaGetLastError();
}

int b200va_stager_add_f32(b200va_stager_t* s, const float* hA, const float* hB, float* hC, size_t n,
                          int variant, int mode)
{
    if (!s || (n && (!hA || !hB || !hC))) return B200VA_ERR_INVALID;
    RC_TRY(check_variant(variant));
    if (mode < B200VA_STAGE_AUTO || mode > B200VA_STAGE_REGISTER) return B200VA_ERR_INVALID;
    DeviceGuard guard(s->device);
    CU_TRY(guard.err);
    const size_t bytes = n * sizeof(float);
    if (mode == B200VA_STAGE_AUTO) {
        const bool pinned = n == 0 || (host_is_pinned(hA) && host_is_pinned(hB) && host_is_pinned(hC));
        mode = pinned ? B200VA_STAGE_LANES : (3 * bytes >= (size_t{8} << 20) ? B200VA_STAGE_REGISTER : B200VA_STAGE_BOUNCE);
    }
    if (mode == B200VA_STAGE_REGISTER) {
        // page-lock the caller's arrays once (outside the timed pipeline: it is a one-off cost of the first call)
        const bool ok = ensure_registered(s, hA, bytes) && ensure_registered(s, hB, bytes) && ensure_registered(s, hC, bytes);
        if (!ok) mode = B200VA_STAGE_BOUNCE;
    }
    s->last_mode = mode;
    CU_TRY(cudaEventRecord(s->ev_start, s->main));
    int rc = B200VA_OK;
    switch (mode) {
        case B200VA_STAGE_ZEROCOPY: rc = stage_zero_copy(s, hA, hB, hC, n, variant); break;
        case B200VA_STAGE_SLOTS:    rc = stage_slots(s, hA, hB, hC, n, variant); break;
        case B200VA_STAGE_LANES:
        case B200VA_STAGE_REGISTER: rc = stage_lanes(s, hA, hB, hC, n, variant); break;
        case B200VA_STAGE_BOUNCE:   rc = stage_bounce(s, hA, hB, hC, n, variant); break;
    }
    if (rc == B200VA_OK) rc = cuda_err(cudaEventRecord(s->ev_stop, s->main));
    if (rc == B200VA_OK) rc = cuda_err(cudaStreamSynchronize(s->main));
    if (rc != B200VA_OK) { stager_drain(s); return rc; }
    CU_TRY(cudaEventElapsedTime(&s->last_ms, s->ev_start, s->ev_stop));
    return B200VA_OK;
}

int b200va_stager_last_ms(b200va_stager_t* s, float* ms)
{
    if (!s || !ms) return B200VA_ERR_INVALID;
    *ms = s->last_ms;
    return B200VA_OK;
}

int b200va_stager_last_mode(b200va_stager_t* s, int* mode)
{
    if (!s || !mode) return B200VA_ERR_INVALID;
    *mode = s->last_mode;
    return B200VA_OK;
}

int b200va_add_f32_host(const float* hA, const float* hB, float* hC, size_t n, int device, int variant)
{
    b200va_stager_t* s = nullptr;
    size_t chunk = size_t{1} << 25;
    if (n < chunk) chunk = n ? n : 1;
    RC_TRY(dev_info(device, nullptr));
    DeviceGuard guard(device);          // cudaPointerGetAttributes below needs a current device; restored on return
    CU_TRY(guard.err);
    // pinned/registered arrays go straight to the copy engines; pageable ones through the bounce pool
    // (one-shot: page-locking 3 arrays for a single pass costs more than bouncing them)
    const bool pageable = n && !(host_is_pinned(hA) && host_is_pinned(hB) && host_is_pinned(hC));
    // pinning the bounce ring costs ~0.35 ms/MiB, so keep it small (9 x 8 MiB)
    if (pageable && chunk > (size_t{1} << 21)) chunk = size_t{1} << 21;
    RC_TRY(b200va_stager_create(&s, device, chunk, n > chunk ? 3 : 1));
    const int rc = b200va_stager_add_f32(s, hA, hB, hC, n, variant, pageable ? B200VA_STAGE_BOUNCE : B200VA_STAGE_LANES);
    b200va_stager_destroy(s);
    return rc;
}
