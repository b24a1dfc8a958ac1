/*
 * i3d_host.h — what every host translation unit of the engine shares: device buffers, the CUDA error check, launch sizes and the
 * phase timers.  No kernels: it includes no .cuh that defines one, so a module that includes it keeps its own device code.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <algorithm>
#include <initializer_list>
#include <map>
#include <string>
#include <vector>

#include "i3d_grid.cuh"

namespace i3d
{

struct CudaError { cudaError_t code; const char* what; const char* file; int line; };

#define CK(call)                                                                  \
    do {                                                                          \
        cudaError_t _e = (call);                                                  \
        if (_e != cudaSuccess) throw ::i3d::CudaError{_e, #call, __FILE__, __LINE__}; \
    } while (0)

template <class T>
struct Dev
{
    T* p = nullptr;
    size_t cap = 0;
    ~Dev() { release(); }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    void ensure(size_t count)
    {
        if (count <= cap) return;
        release();
        CK(cudaMalloc(&p, std::max<size_t>(count, 1) * sizeof(T)));
        cap = count;
    }
    void swap(Dev& o) { std::swap(p, o.p); std::swap(cap, o.cap); }
};

inline unsigned blocks_for(size_t n, int threads = kThreads) { return static_cast<unsigned>((n + threads - 1) / threads); }

// ---- phase and kernel timers ------------------------------------------------------------------
struct Phase { double ms = 0.0; int64_t count = 0; };

// The engine's timing state: the event pool, the event pairs of the current call (resolved by collect_kernel_times), the phase table
// i3d_phase_ms / i3d_phase_count read, and the timer level (0: phases + the roofline kernels; 1: every kernel of the iteration, set by
// i3d_debug_set_kernel_timers; -1: nothing is recorded)
struct Timing
{
    std::vector<cudaEvent_t> pool;
    struct Pair { int a, b; const char* name; };
    std::vector<Pair> pending;
    size_t used = 0;
    std::map<std::string, Phase> phases;
    int level = 0;
};

// Brackets stream work (a phase, or one kernel launch) with two events from the pool; resolved without extra synchronisation by
// collect_kernel_times().  `level` 0 = always recorded: the phases and the roofline kernels (k_eg_rows, k_eg_apply, k_select_obs);
// level 1 = only when i3d_debug_set_kernel_timers(e, 1) asked for the per-kernel table.  (An event record between two kernels makes
// the second one wait for the first one's completion the ordinary way: no programmatic overlap across it.)
struct Timer
{
    Timing& tm; cudaStream_t st; int a = -1, b = -1; const char* name;
    Timer(Timing& timing, cudaStream_t stream, const char* nm, int level = 0) : tm(timing), st(stream), name(nm)
    {
        if (level <= tm.level && tm.used + 2 <= tm.pool.size()) { a = static_cast<int>(tm.used++); b = static_cast<int>(tm.used++); cudaEventRecord(tm.pool[a], st); }
    }
    void stop()
    {
        if (a >= 0) { cudaEventRecord(tm.pool[b], st); tm.pending.push_back({a, b, name}); a = -1; }
    }
    ~Timer() { stop(); }
};

// Starts the timing of one call: the event pool is free again, and the phases the call owns start from zero
inline void begin_timing(Timing& tm, std::initializer_list<const char*> owned)
{
    tm.pending.clear(); tm.used = 0;
    for (const char* nm : owned) tm.phases.erase(nm);
}

// Synchronises the stream and adds the time of every pending pair to its phase
inline void collect_kernel_times(Timing& tm, cudaStream_t st)
{
    cudaStreamSynchronize(st);
    for (const auto& t : tm.pending)
    {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, tm.pool[t.a], tm.pool[t.b]) == cudaSuccess) { Phase& p = tm.phases[t.name]; p.ms += ms; p.count += 1; }
    }
    tm.pending.clear(); tm.used = 0;
}

} // namespace i3d
