/*
 * i3d_engine.cu — host side of the H100 joint-refinement engine + the C-ABI of include/i3d_c_api.h.
 *
 * One I3DEngine = one GPU.  i3d_gn_iteration() is one outer iteration of Optimizer::optimize
 * (libintrinsic3d/src/refinement/optimizer.cpp:119-171): observation selection (k_select_obs),
 * residual/Jacobian build (k_eg_rows<ROWS_BUILD>, k_reg_build), weight normalisation + parameter fixing
 * (k_finish_problem), and the Ceres-equivalent LM step: block-Jacobi preconditioned CGNR
 * (k_cg_dir4 / k_eg_apply / k_op_partial / k_cg_update, device-resident scalars), model-cost-change, candidate
 * evaluation (k_eg_rows<ROWS_COST> / k_reg_cost) and the accept/reject decision (k_lm_decide) — the host reads one result struct per trial.
 *
 * No CPU fallback: every entry point that computes fails if the CUDA device is unavailable.
 */
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/i3d_c_api.h"
#include "i3d_kernels.cuh"
#include "i3d_lighting.cuh"
#include "i3d_recolor.cuh"
#include "i3d_gridops.cuh"

using namespace i3d;

#define I3D_ABI_VERSION 1

namespace
{
std::string g_create_error;

// ---- NCCL, bound at run time (dlopen) so that the library has no link-time dependency and shares the NCCL that
// the host process (e.g. torch.distributed) already loaded.  Only ncclAllReduce(sum) is used on the data path.
struct NcclApi
{
    typedef struct { char internal[128]; } UniqueId;
    typedef void* Comm;
    int (*GetUniqueId)(UniqueId*) = nullptr;
    int (*CommInitRank)(Comm*, int, UniqueId, int) = nullptr;
    int (*CommDestroy)(Comm) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, Comm, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    void* handle = nullptr;
    bool load(std::string* err)
    {
        if (handle) return true;
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* nm : names) { handle = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (handle) break; }
        if (!handle) { *err = std::string("cannot dlopen libnccl.so.2: ") + dlerror(); return false; }
        GetUniqueId = reinterpret_cast<decltype(GetUniqueId)>(dlsym(handle, "ncclGetUniqueId"));
        CommInitRank = reinterpret_cast<decltype(CommInitRank)>(dlsym(handle, "ncclCommInitRank"));
        CommDestroy = reinterpret_cast<decltype(CommDestroy)>(dlsym(handle, "ncclCommDestroy"));
        AllReduce = reinterpret_cast<decltype(AllReduce)>(dlsym(handle, "ncclAllReduce"));
        GetErrorString = reinterpret_cast<decltype(GetErrorString)>(dlsym(handle, "ncclGetErrorString"));
        if (!GetUniqueId || !CommInitRank || !CommDestroy || !AllReduce || !GetErrorString) { *err = "libnccl.so.2 lacks required symbols"; return false; }
        return true;
    }
};
NcclApi g_nccl;
enum { NCCL_UINT8 = 1, NCCL_FLOAT32 = 7, NCCL_FLOAT64 = 8, NCCL_SUM = 0 };

struct CudaError { cudaError_t code; const char* what; int line; };
struct NcclError { int code; int line; };

#define CK(call)                                                                  \
    do {                                                                          \
        cudaError_t _e = (call);                                                  \
        if (_e != cudaSuccess) throw CudaError{_e, #call, __LINE__};              \
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

enum Site { SITE_BUILD = 0, SITE_REG, SITE_FINISH, SITE_EG_APPLY, SITE_OP_POST, SITE_UPDATE, SITE_CAND, SITE_EG_COST, SITE_REG_COST, SITE_COUNT };
constexpr int kSiteVals = 9;

struct Phase { double ms = 0.0; int64_t count = 0; };
} // namespace

struct I3DEngine
{
    int device = 0;
    cudaStream_t stream = nullptr;
    std::string error;

    // grid
    int64_t n = 0;
    float voxel_size = 0.f, truncation = 0.f;
    Dev<int32_t> x, y, z, nbr;
    Dev<double> sdf0, sdfA, albA, sdfB, albB, sh;
    Dev<float> weight;
    Dev<uchar4> rgb;
    double* sdf = nullptr; double* alb = nullptr;       // current state
    double* c_sdf = nullptr; double* c_alb = nullptr;   // candidate
    bool have_sh = false;
    // frames
    int F = 0, W = 0, H = 0;
    double pyr_scale = 1.0;
    Dev<float> lum, depth;
    Dev<float> tile_min, tile_max;
    Dev<unsigned long long> cull_stats;   // per-frame 32x32 depth tiles for the conservative frame culling of k_select_obs
    // camera
    Dev<double> camA, camB;
    double* cam = nullptr; double* c_cam = nullptr;
    bool have_cam = false;
    // per-iteration
    Dev<uint8_t> flags;
    // upload scratch kept across calls (cudaMalloc/cudaFree per upload would serialise the device)
    Dev<int32_t> up_xyz, up_vals; Dev<uint8_t> up_rgb; Dev<unsigned long long> up_keys; Dev<int> up_dup; Dev<double> up_sh;
    uint64_t hash_cap = 0;     // capacity (power of two) of the device hash table up_keys/up_vals of the CURRENT grid
    // second set of voxel arrays: pruning / upsampling write into it and swap (no cudaMalloc / cudaFree per call once it has grown)
    Dev<int32_t> sp_x, sp_y, sp_z; Dev<double> sp_sdf0, sp_sdf, sp_alb; Dev<float> sp_w; Dev<uchar4> sp_rgb;
    Dev<int32_t> act, scan_counts, scan_total;
    int n_active = 0, K = 0, stride = 0;
    Dev<float> Rt;
    Dev<FramePose> pose_ctx, pose_ctx_c;
    Dev<int32_t> obs_frame, row_frame;
    Dev<float> obs_w, J, row_w;
    Dev<double> row_res, row_wraw;
    Dev<float> ea_w;
    Dev<double> lap;
    Dev<float> cam_acc;
    Dev<double> minv, type_w;
    Dev<int> fail_flag;
    // vectors
    Dev<float> v_bg, v_cg, v_s, v_jtj, v_b, v_x, v_r, v_z, v_p, v_ps, v_qg, v_tr, v_delta;
    Dev<double> v_bgd, v_cgd, v_qgd, cam_accd;     // double accumulators of k_eg_accum / k_eg_apply
    Dev<CgCtl> ctl;
    // reductions
    Dev<double> red_partials, red_out;
    Dev<unsigned int> red_counters;
    size_t max_blocks = 0;
    // debug
    bool keep_raw = false;
    Dev<float> dbg_v;            // input vector of i3d_debug_apply_operator
    I3DParams last_params{};
    bool have_iter = false;
    std::map<std::string, Phase> phases;
    cudaEvent_t ev[16];
    // per-kernel timing (CUDA events on the launching stream) for the two roofline kernels
    std::vector<cudaEvent_t> ev_pool;
    struct TimedLaunch { int a, b; const char* name; };
    std::vector<TimedLaunch> timed;
    size_t ev_used = 0;
    int64_t launches = 0;        // kernels launched during the last i3d_gn_iteration
    int64_t host_syncs = 0;      // cudaStreamSynchronize calls of the last i3d_gn_iteration
    int timer_level = 0;         // 0: phases + the roofline kernels (sampled); 1: every kernel of the iteration (i3d_debug_set_kernel_timers)
    Dev<IterDev> iter_dev;       // device-resident result / LM state of the current iteration
    int last_cg_iterations = 4, prev_cg_iterations = 4;  // PCG iteration counts of the previous two solves: their maximum sizes the first launch batch
    // colour frames for the recolouring pass (i3d_recolor.cuh)
    Dev<uint8_t> color;
    bool have_color = false;
    Dev<unsigned long long> recolor_counts;
    // SVSH lighting (i3d_lighting.cuh)
    Dev<int32_t> sv_table, sv_index, sv_nbr;
    Dev<int> sv_scalars, sv_deg;       // sv_scalars: [0..5] index bounds, [6] subvolume count
    Dev<double> sv_acc, sv_work;
    Dev<I3DLightingInfo> sv_info;
    Dev<uint8_t> sh_has;
    int sv_S = 0;
    double* sv_x = nullptr;            // [S][9] subvolume SH of the last estimate (inside sv_work)
    // shard (multi-GPU)
    int64_t shard_begin = 0, shard_end = -1;
    int rank = 0, world = 1;
    NcclApi::Comm comm = nullptr;
    bool shard_ready = false;
    Dev<uint8_t> held;             // [2n] bit0 held, bit1 shared
    Dev<uint8_t> held_mask;        // [2n] 0/1
    Dev<int32_t> slist;
    int64_t n_shared = 0;
    int64_t hv0 = 0, hv1 = 0;             // index hull of the voxels whose unknowns this rank holds
    int64_t loc_begin = 0, loc_end = 0;   // index range of the voxels this rank reads per-iteration data of (own + 4 stencil rings)
    Dev<double> xbuf;
    // peer-memory exchange (mailbox mapped into every peer with CUDA IPC; see k_xchg_pull)
    Dev<uint8_t> mbox;
    size_t mbox_cap = 0;               // doubles per buffer
    bool p2p_ready = false;
    unsigned int xseq = 0;             // sequence number of the last exchange (identical on every rank)
    std::vector<void*> peer_base;      // [world] mapped mailbox bases (own entry = mbox.p)
    Dev<double*> d_peer_data;
    Dev<unsigned int*> d_peer_flags;
    static constexpr size_t kMboxFlagBytes = 4096;
    P2PView p2p_view() const { P2PView v; v.rank = rank; v.world = world; v.peer_data = d_peer_data.p; v.peer_flags = d_peer_flags.p; v.cap = mbox_cap; return v; }
    Shard shard() const
    {
        Shard sh;
        if (world > 1) { sh.own_begin = shard_begin; sh.own_end = shard_end; sh.hv0 = hv0; sh.hv1 = hv1; sh.cam_owner = (rank == 0); sh.defer = 1; sh.loc_begin = loc_begin; sh.loc_end = loc_end; }
        else { sh.own_begin = 0; sh.own_end = n; sh.hv0 = 0; sh.hv1 = n; sh.cam_owner = 1; sh.defer = 0; sh.loc_begin = 0; sh.loc_end = n; }
        return sh;
    }
    int64_t held_count() const { return (world > 1 ? 2 * (hv1 - hv0) : 2 * n) + 6 * static_cast<int64_t>(F) + 9; }
    ShareView share_view() const { ShareView v; v.n_shared = n_shared; v.slist = slist.p; v.held = held_mask.p; return v; }

    int64_t U() const { return 2 * n + 6 * static_cast<int64_t>(F) + 9; }
    ReduceSite site(int s)
    {
        ReduceSite r;
        r.partials = red_partials.p + static_cast<size_t>(s) * max_blocks * kSiteVals;
        r.counter = red_counters.p + s;
        r.out = red_out.p + s * kSiteVals;
        return r;
    }
    GridView grid_view(const double* sdf_ptr, const double* alb_ptr) const
    {
        GridView g;
        g.n = n; g.x = x.p; g.y = y.p; g.z = z.p; g.sdf0 = sdf0.p; g.sdf = sdf_ptr; g.albedo = alb_ptr; g.weight = weight.p; g.rgb = rgb.p;
        g.nbr = nbr.p; g.sh = sh.p; g.voxel_size = voxel_size; g.truncation = truncation;
        return g;
    }
    FrameView frame_view() const { FrameView f; f.F = F; f.W = W; f.H = H; f.lum = lum.p; f.depth = depth.p; f.pyr_scale = pyr_scale; return f; }
};

namespace
{

int fail(I3DEngine* e, const char* fmt, ...)
{
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    if (e) e->error = buf; else g_create_error = buf;
    return 1;
}

template <class Fn>
int guarded(I3DEngine* e, Fn&& fn)
{
    try
    {
        if (e) CK(cudaSetDevice(e->device));
        return fn();
    }
    catch (const CudaError& ce)
    {
        return fail(e, "CUDA error %d (%s) at i3d_engine.cu:%d: %s", static_cast<int>(ce.code), cudaGetErrorString(ce.code), ce.line, ce.what);
    }
    catch (const NcclError& ne) { return fail(e, "NCCL error %d (%s) at i3d_engine.cu:%d", ne.code, g_nccl.GetErrorString ? g_nccl.GetErrorString(ne.code) : "?", ne.line); }
    catch (const std::exception& ex) { return fail(e, "exception: %s", ex.what()); }
}

// Device hash table (coordinates -> voxel index) and the 12-entry neighbour table of the grid in e->x/y/z; replaces every
// unordered_map::find of SparseVoxelGrid on the path.  Returns non-zero if two voxels share coordinates.
int rebuild_topology(I3DEngine* e)
{
    cudaStream_t st = e->stream;
    const int64_t n = e->n;
    e->nbr.ensure(static_cast<size_t>(NB_COUNT) * n);
    uint64_t cap = 1; while (cap < static_cast<uint64_t>(2 * n)) cap <<= 1;
    e->up_keys.ensure(cap); e->up_vals.ensure(cap); e->up_dup.ensure(1);
    e->hash_cap = cap;
    CK(cudaMemsetAsync(e->up_keys.p, 0xFF, cap * sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(e->up_dup.p, 0, sizeof(int), st));
    k_hash_insert<<<blocks_for(n), kThreads, 0, st>>>(n, e->x.p, e->y.p, e->z.p, e->up_keys.p, e->up_vals.p, cap - 1, e->up_dup.p);
    k_build_nbr<<<blocks_for(n), kThreads, 0, st>>>(n, e->x.p, e->y.p, e->z.p, e->up_keys.p, e->up_vals.p, cap - 1, e->nbr.p);
    int hdup = 0;
    CK(cudaMemcpyAsync(&hdup, e->up_dup.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    return hdup;
}

// installs freshly built voxel arrays (count m) as the engine's grid and rebuilds the topology; everything derived from the old
// voxel set (per-voxel SH, shard, last iteration) is invalidated
int install_grid(I3DEngine* e, int64_t m, Dev<int32_t>& x, Dev<int32_t>& y, Dev<int32_t>& z, Dev<double>& sdf0, Dev<double>& sdf, Dev<double>& alb,
                 Dev<float>& weight, Dev<uchar4>& rgb)
{
    e->x.swap(x); e->y.swap(y); e->z.swap(z); e->sdf0.swap(sdf0); e->sdfA.swap(sdf); e->albA.swap(alb); e->weight.swap(weight); e->rgb.swap(rgb);
    e->n = m;
    e->sdfB.ensure(static_cast<size_t>(m)); e->albB.ensure(static_cast<size_t>(m));
    e->sdf = e->sdfA.p; e->c_sdf = e->sdfB.p; e->alb = e->albA.p; e->c_alb = e->albB.p;
    e->have_sh = false; e->have_iter = false; e->shard_ready = false; e->sv_S = 0; e->sv_x = nullptr;
    if (e->world > 1) { e->shard_begin = 0; e->shard_end = -1; }
    return rebuild_topology(e);
}

void ensure_reduction_scratch(I3DEngine* e)
{
    const size_t elems = std::max<size_t>(static_cast<size_t>(e->U()), static_cast<size_t>(e->n) * I3D_MAX_OBS * 4 + 256);
    const size_t need = blocks_for(elems) + 8;
    if (need > e->max_blocks || !e->red_partials.p)
    {
        e->max_blocks = need;
        e->red_partials.ensure(static_cast<size_t>(SITE_COUNT) * need * kSiteVals);
        e->red_out.ensure(SITE_COUNT * kSiteVals);
        e->red_counters.ensure(SITE_COUNT);
        CK(cudaMemsetAsync(e->red_counters.p, 0, SITE_COUNT * sizeof(unsigned int), e->stream));
        CK(cudaMemsetAsync(e->red_out.p, 0, SITE_COUNT * kSiteVals * sizeof(double), e->stream));
    }
}

void ensure_vectors(I3DEngine* e)
{
    const size_t U = static_cast<size_t>(e->U());
    Dev<float>* vs[] = {&e->v_bg, &e->v_cg, &e->v_s, &e->v_jtj, &e->v_b, &e->v_x, &e->v_r, &e->v_z, &e->v_p, &e->v_ps, &e->v_qg, &e->v_delta};
    for (auto* v : vs) v->ensure(U);
    Dev<double>* vd[] = {&e->v_bgd, &e->v_cgd, &e->v_qgd};
    for (auto* v : vd) v->ensure(U);
    e->cam_accd.ensure(CamAccLayout{e->F}.size());
    e->v_tr.ensure(static_cast<size_t>(e->n));
    e->ctl.ensure(1);
    e->minv.ensure(36 * static_cast<size_t>(e->F) + 41);
    e->type_w.ensure(4);
    e->fail_flag.ensure(1);
    e->cam_acc.ensure(CamAccLayout{e->F}.size());
    ensure_reduction_scratch(e);
}

SolveVecs solve_vecs(I3DEngine* e)
{
    SolveVecs sv;
    sv.n = e->n; sv.F = e->F; sv.U = e->U();
    sv.bg = e->v_bg.p; sv.cg = e->v_cg.p; sv.s = e->v_s.p; sv.jtj = e->v_jtj.p; sv.b = e->v_b.p;
    sv.x = e->v_x.p; sv.r = e->v_r.p; sv.z = e->v_z.p; sv.p = e->v_p.p; sv.ps = e->v_ps.p; sv.qg = e->v_qg.p; sv.qgd = e->v_qgd.p; sv.tr = e->v_tr.p;
    return sv;
}

// brackets one kernel launch with two events from the pool; resolved by collect_kernel_times()
// (an event record between two kernels makes the second one wait for the first one's completion the ordinary way: no programmatic
// overlap across it.  `level` 0 = always timed: the two roofline kernels (k_eg_rows, k_eg_apply) and k_select_obs; level 1 = only when i3d_debug_set_kernel_timers(e, 1) asked for the per-kernel table.)
struct KernelTimer
{
    I3DEngine* e; int a = -1, b = -1; const char* name;
    KernelTimer(I3DEngine* eng, const char* nm, int level = 1) : e(eng), name(nm)
    {
        if (level > e->timer_level) return;
        if (e->ev_used + 2 <= e->ev_pool.size()) { a = static_cast<int>(e->ev_used++); b = static_cast<int>(e->ev_used++); cudaEventRecord(e->ev_pool[a], e->stream); }
    }
    ~KernelTimer()
    {
        if (a >= 0) { cudaEventRecord(e->ev_pool[b], e->stream); e->timed.push_back({a, b, name}); }
    }
};

void collect_kernel_times(I3DEngine* e)
{
    cudaStreamSynchronize(e->stream);
    for (const auto& t : e->timed)
    {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, e->ev_pool[t.a], e->ev_pool[t.b]) == cudaSuccess) { Phase& p = e->phases[t.name]; p.ms += ms; p.count += 1; }
    }
    e->timed.clear(); e->ev_used = 0;
    e->phases["launches"].count = e->launches;
    e->phases["host_syncs"].count = e->host_syncs;
}

// phase timer: two events from the pool, resolved (without extra synchronisation) by collect_kernel_times()
struct Timer
{
    I3DEngine* e; int a = -1, b = -1; const char* name; bool stopped = false;
    Timer(I3DEngine* eng, const char* nm, int /*slot*/) : e(eng), name(nm)
    {
        if (e->ev_used + 2 <= e->ev_pool.size()) { a = static_cast<int>(e->ev_used++); b = static_cast<int>(e->ev_used++); cudaEventRecord(e->ev_pool[a], e->stream); }
    }
    void stop()
    {
        if (stopped) return;
        stopped = true;
        if (a >= 0) { cudaEventRecord(e->ev_pool[b], e->stream); e->timed.push_back({a, b, name}); }
    }
    ~Timer() { stop(); }
};

#define NK(call)                                                            \
    do {                                                                    \
        int _r = (call);                                                    \
        if (_r != 0) throw NcclError{_r, __LINE__};                         \
    } while (0)


// Every kernel of the Gauss-Newton iteration is launched with programmatic stream serialization (programmatic dependent launch):
// the kernels begin with griddepcontrol.wait (pdl_prologue(), i3d_kernels.cuh), so the next grid's launch latency overlaps the tail
// of its predecessor instead of following it.  I3D_PDL=0 disables the attribute (the device-side wait is then a no-op).
template <class... KArgs, class... Args>
void pdl_launch(I3DEngine* e, void (*kern)(KArgs...), unsigned grid, unsigned block, size_t smem, Args&&... args)
{
    static const bool enabled = [] { const char* v = std::getenv("I3D_PDL"); return !(v && v[0] == '0'); }();
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = e->stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = enabled ? 1 : 0;
    CK(cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...));
}

// k_eg_rows variant selection.  Cost evaluation (ROWS_COST): the pose table of all F frames is staged into shared memory by a bulk-async
// copy (256 threads, 2 blocks per SM) when two blocks with their per-voxel state and the table fit into the SM's shared memory —
// measured at C3: 0.455 ms staged vs 0.486 ms from L1.  Jacobian build (ROWS_BUILD): 128 threads x 4 blocks, poses from L1 — the
// staged variant was SLOWER there (0.800 vs 0.719 ms: the 40-float derivative state per thread makes the 256-thread blocks 108 KB
// each, and the block-granular tail costs more than the L1 misses it removes).  profiles/r02p_*.json; I3D_ROWS_STAGE=0 / 2 force none / both.
template <int MODE>
void launch_eg_rows(I3DEngine* e, const GridView& g, const CamView& cv, const EgRows& rows, const int32_t* obs_frame, const float* obs_w)
{
    static const int stage_mode = [] { const char* v = std::getenv("I3D_ROWS_STAGE"); return !I3D_ROWS_STAGE_POSE ? 0 : (v ? std::atoi(v) : 1); }();
    const size_t smem_stage = rows_smem_bytes(MODE, 256, true, e->F);
    const bool stage = (stage_mode == 2 || (stage_mode == 1 && MODE == ROWS_COST)) && 2 * (smem_stage + 1024) <= 227u * 1024u;
    if (stage)
    {
        auto kern = k_eg_rows<MODE, 256, true>;
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_stage)));
        pdl_launch(e, kern, blocks_for(static_cast<size_t>(rows.stride), 256), 256, smem_stage, g, e->frame_view(), cv, rows, obs_frame, obs_w, e->site(SITE_EG_COST));
    }
    else
    {
        auto kern = k_eg_rows<MODE, 128, false>;
        const size_t smem = rows_smem_bytes(MODE, 128, false, e->F);
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        pdl_launch(e, kern, blocks_for(static_cast<size_t>(rows.stride), 128), 128, smem, g, e->frame_view(), cv, rows, obs_frame, obs_w, e->site(SITE_EG_COST));
    }
}

// in-place sum over ranks of `count` (<= 30) doubles living on the device, optionally followed by the scalar epilogue `kind`
// (EPI_*; -1 = none) that consumes them.  Peer-memory path: ONE single-warp launch (k_xchg_scalars); NCCL path: ncclAllReduce
// + k_epilogue.  No-op on a single GPU.
void allreduce_scalars(I3DEngine* e, double* dev, int count, int kind, int respect_done)
{
    if (e->world <= 1) return;
    if (e->p2p_ready && count <= 30)
    {
        const unsigned int seq = ++e->xseq;
        pdl_launch(e, k_xchg_scalars, 1, 32, 0, e->p2p_view(), seq, dev, count, e->ctl.p, kind, respect_done);
        e->launches += 1;
        return;
    }
    NK(g_nccl.AllReduce(dev, dev, static_cast<size_t>(count), NCCL_FLOAT64, NCCL_SUM, e->comm, e->stream));
    if (kind >= 0) { pdl_launch(e, k_epilogue, 1, 32, 0, e->ctl.p, dev, kind, respect_done); e->launches += 1; }
}

// Multi-GPU exchange after a partial accumulation: [v0 | v1 | extra floats | extra doubles] at the shared unknowns are packed
// and summed over ranks — by pulling the peers' packed buffers over NVLink (k_xchg_pull), or with ONE ncclAllReduce when the
// peer mailboxes are not connected — and written back.
void exchange(I3DEngine* e, float* v0, float* v1, float* extra_f, int n_extra_f, double* extra_d, int n_extra_d, int respect_done, int epilogue_kind = -1)
{
    if (e->world <= 1) return;
    const ShareView shv = e->share_view();
    const size_t nv = v1 ? 2 : 1;
    const size_t total = nv * static_cast<size_t>(e->n_shared) + n_extra_f + n_extra_d;
    const size_t threads = static_cast<size_t>(e->n_shared) + n_extra_f + n_extra_d;
    if (e->p2p_ready && total <= e->mbox_cap)
    {
        const unsigned int seq = ++e->xseq;
        double* buf = reinterpret_cast<double*>(e->mbox.p + I3DEngine::kMboxFlagBytes) + static_cast<size_t>(seq & 1u) * e->mbox_cap;
        pdl_launch(e, k_pack, blocks_for(threads), kThreads, 0, shv, v0, v1, extra_f, n_extra_f, extra_d, n_extra_d, buf, e->ctl.p, respect_done);
        pdl_launch(e, k_xchg_pull, blocks_for(threads), kThreads, 0, e->p2p_view(), seq, shv, v0, v1, extra_f, n_extra_f, extra_d, n_extra_d, e->ctl.p, respect_done, epilogue_kind);
        e->launches += 2;
        return;
    }
    e->xbuf.ensure(2 * static_cast<size_t>(e->n_shared) + CamAccLayout{e->F}.size() + 64);
    pdl_launch(e, k_pack, blocks_for(threads), kThreads, 0, shv, v0, v1, extra_f, n_extra_f, extra_d, n_extra_d, e->xbuf.p, e->ctl.p, respect_done);
    NK(g_nccl.AllReduce(e->xbuf.p, e->xbuf.p, total, NCCL_FLOAT64, NCCL_SUM, e->comm, e->stream));
    pdl_launch(e, k_unpack, blocks_for(threads), kThreads, 0, shv, v0, v1, extra_f, n_extra_f, extra_d, n_extra_d, e->xbuf.p, e->ctl.p, respect_done);
    e->launches += 2;
    if (epilogue_kind >= 0) { pdl_launch(e, k_epilogue, 1, 32, 0, e->ctl.p, extra_d, epilogue_kind, respect_done); e->launches += 1; }
}

size_t apply_smem_bytes(int F, int K)
{
    return static_cast<size_t>((6 * F + 9 + 15) & ~15) * sizeof(double) + static_cast<size_t>(K) * 6 * kThreads * sizeof(float);
}

size_t accum_smem_bytes(int F, int K)
{
    return static_cast<size_t>((CamAccLayout{F}.size() + 15) & ~15) * sizeof(double) + static_cast<size_t>(K) * 8 * kThreads * sizeof(float);
}

// The per-frame camera accumulators of k_eg_accum and k_eg_apply live in one block's shared memory: refuse, before anything is
// launched, a frame count whose dynamic plus static shared memory exceeds the device's opt-in limit per block.
int check_frame_limit(I3DEngine* e, int F, int K)
{
    int optin = 0;
    CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, e->device));
    cudaFuncAttributes fa_acc{}, fa_app{};
    CK(cudaFuncGetAttributes(&fa_acc, k_eg_accum));
    CK(cudaFuncGetAttributes(&fa_app, k_eg_apply<APPLY_CG>));
    const size_t lim = static_cast<size_t>(optin);
    auto fits = [&](int f) { return fa_acc.sharedSizeBytes + accum_smem_bytes(f, K) <= lim && fa_app.sharedSizeBytes + apply_smem_bytes(f, K) <= lim; };
    if (fits(F)) return 0;
    int fmax = 0;
    while (fits(fmax + 1)) ++fmax;
    return fail(e, "i3d_gn_iteration: %d frames at K = %d observations need %zu bytes of shared memory per block in k_eg_accum (device limit %d): "
                   "at most %d frames at K = %d", F, K, fa_acc.sharedSizeBytes + accum_smem_bytes(F, K), optin, fmax, K);
}

// applies the CGNR operator to the vector whose Jacobi-scaled copy is in sv.ps: afterwards qg holds the (globally summed)
// raw J'^T J' part; k_cg_update forms q = s*qg + D^2 v on the fly and resets qg.
void launch_operator(I3DEngine* e, const GridView& g, const RegView& rv, const EgRows& rows, const SolveVecs& sv, const Shard& sh, const float* vin,
                     float dmin, float dmax, int is_cg_iteration, bool sample_timing = false)
{
    if (rows.n_active > 0)
    {
        KernelTimer kt(e, "k_eg_apply", 0);     // the dominant kernel: every launch is timed (roofline = true average)
        pdl_launch(e, k_eg_apply<APPLY_CG>, blocks_for(rows.n_active), kThreads, apply_smem_bytes(e->F, rows.K), g, rows, rv, sv, sv.ps, e->ctl.p, 1, e->site(SITE_EG_APPLY));
    }
    e->launches += 2;
    {
        KernelTimer kt(e, "k_op_partial");
        pdl_launch(e, (k_op_partial<APPLY_CG, 4>), blocks_for(static_cast<size_t>((e->held_count() + 3) / 4)), kThreads, 0, 
            g, rv, sv, sh, e->held_count(), vin, sv.ps, e->type_w.p, dmin, dmax, e->ctl.p, 1, e->site(SITE_OP_POST), e->site(SITE_EG_APPLY).out, is_cg_iteration);
    }
    if (e->world > 1)
    {
        KernelTimer kt(e, "exchange");
        exchange(e, sv.qg, nullptr, sv.qg + 2 * e->n, 6 * e->F + 9, e->site(SITE_OP_POST).out, 1, 1, is_cg_iteration ? EPI_OPERATOR_CG : -1);
    }
}

// One outer Gauss-Newton iteration.  Host synchronisations: ONE after the activity scan (row count -> launch sizes) and ONE
// per LM trial (the device-resident IterDev struct comes back; typically a single trial), plus one per extra PCG batch when a
// solve needs more iterations than the previous one did.  Everything else — type weights, Jacobi scaling, PCG scalars, the
// TrustRegionMinimizer accept/reject logic and the radius update — is decided on the device (k_type_weights, k_iter_finish,
// k_lm_begin, k_lm_decide).
int gn_iteration_impl(I3DEngine* e, const I3DParams& P, I3DIterInfo& info)
{
    std::memset(&info, 0, sizeof(info));
    if (e->n <= 0) return fail(e, "i3d_gn_iteration: no grid uploaded");
    if (e->F <= 0) return fail(e, "i3d_gn_iteration: no frames uploaded");
    if (!e->have_cam) return fail(e, "i3d_gn_iteration: camera not set");
    if (!e->have_sh) return fail(e, "i3d_gn_iteration: SH coefficients not set");
    if (e->world > 1 && !e->shard_ready) return fail(e, "i3d_gn_iteration: world > 1 but i3d_set_shard was not called after the grid/frames upload");
    int K = P.num_observations;
    if (K <= 0 || K > e->F) K = e->F;
    if (K > I3D_MAX_OBS) return fail(e, "i3d_gn_iteration: num_observations (%d) exceeds I3D_MAX_OBS (%d)", K, I3D_MAX_OBS);
    if (P.lm_steps < 1) return fail(e, "i3d_gn_iteration: lm_steps < 1");
    if (P.residual_reset_period < 1) return fail(e, "i3d_gn_iteration: residual_reset_period < 1");
    if (check_frame_limit(e, e->F, K) != 0) return 1;
    e->K = K;
    e->last_params = P;
    e->phases.clear(); e->timed.clear(); e->ev_used = 0; e->launches = 0; e->host_syncs = 0;
    const int64_t n = e->n;
    const int F = e->F;
    const bool multi = e->world > 1;
    cudaStream_t st = e->stream;
    ensure_vectors(e);
    e->iter_dev.ensure(1);
    const Shard sh = e->shard();
    const int64_t own = sh.own_end - sh.own_begin;
    const int64_t hc = e->held_count();
    const size_t U = static_cast<size_t>(e->U());
    Timer t_total(e, "total", 0);
    auto sync = [&]() { CK(cudaStreamSynchronize(st)); e->host_syncs += 1; };

    // ------------------------------------------------------------------ activity, compaction of the rows this rank owns
    Timer t_sel(e, "select", 1);
    e->flags.ensure(n);
    GridView g = e->grid_view(e->sdf, e->alb);
    // flags over the range this rank reads (own voxels + 4 stencil rings); compaction of the owned rows over the owned range
    pdl_launch(e, k_flags, blocks_for(static_cast<size_t>(sh.loc_end - sh.loc_begin)), kThreads, 0, g, sh, P.thres_shell, P.fix_all_albedo, e->flags.p);
    const int nscan = std::max(1, static_cast<int>((own + kScanChunk - 1) / kScanChunk));
    e->scan_counts.ensure(nscan); e->scan_total.ensure(1); e->act.ensure(n);
    pdl_launch(e, k_scan_count, nscan, kThreads, 0, own, e->flags.p + sh.own_begin, FL_ROW, e->scan_counts.p);
    pdl_launch(e, k_scan_blocks, 1, 1024, 0, nscan, e->scan_counts.p, e->scan_total.p);
    pdl_launch(e, k_scan_scatter, nscan, kThreads, 0, own, e->flags.p + sh.own_begin, FL_ROW, e->scan_counts.p, e->act.p, static_cast<int32_t>(sh.own_begin));
    e->launches += 4;
    // while the scan runs: everything that does not depend on the row count
    const CamAccLayout lay{F};
    CK(cudaMemsetAsync(e->v_bg.p, 0, U * sizeof(float), st));
    CK(cudaMemsetAsync(e->v_cg.p, 0, U * sizeof(float), st));
    CK(cudaMemsetAsync(e->v_qg.p, 0, U * sizeof(float), st));
    CK(cudaMemsetAsync(e->v_delta.p, 0, U * sizeof(float), st));
    CK(cudaMemsetAsync(e->v_tr.p, 0, static_cast<size_t>(n) * sizeof(float), st));      // E_r row values: only active ring voxels are written (k_eg_apply)
    CK(cudaMemsetAsync(e->cam_acc.p, 0, lay.size() * sizeof(float), st));
    CK(cudaMemsetAsync(e->v_bgd.p, 0, U * sizeof(double), st));
    CK(cudaMemsetAsync(e->v_cgd.p, 0, U * sizeof(double), st));
    CK(cudaMemsetAsync(e->v_qgd.p, 0, U * sizeof(double), st));
    CK(cudaMemsetAsync(e->cam_accd.p, 0, lay.size() * sizeof(double), st));
    CK(cudaMemsetAsync(e->red_out.p, 0, 2 * kSiteVals * sizeof(double), st));   // SITE_BUILD, SITE_REG (a rank without rows skips the kernels)
    e->Rt.ensure(12 * static_cast<size_t>(F));
    e->pose_ctx.ensure(F); e->pose_ctx_c.ensure(F);
    pdl_launch(e, k_pose_mats, blocks_for(F, 64), 64, 0, F, e->cam, e->Rt.p);
    pdl_launch(e, k_frame_pose, blocks_for(F, 64), 64, 0, F, e->cam, e->pose_ctx.p);
    e->launches += 2;
    int32_t n_active = 0;
    double hc9[9];
    CK(cudaMemcpyAsync(&n_active, e->scan_total.p, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    // intrinsics * pyr_scale cast to float (optimizer.cpp:124-127; Camera::setIntrinsics)
    CK(cudaMemcpyAsync(hc9, e->cam + 6 * static_cast<size_t>(F), 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
    sync();
    e->n_active = n_active;
    const int stride = (n_active + 63) & ~63;          // slots per k: keeps every J column segment 256 B aligned
    e->stride = stride;
    const size_t S = static_cast<size_t>(K) * stride;

    // ------------------------------------------------------------------ k1 observation selection
    e->obs_frame.ensure(S + 1); e->obs_w.ensure(S + 1);
    if (n_active > 0)
    {
        SelectCam sc;
        sc.fx = static_cast<float>(hc9[0] * e->pyr_scale); sc.fy = static_cast<float>(hc9[1] * e->pyr_scale);
        sc.cx = static_cast<float>(hc9[2] * e->pyr_scale); sc.cy = static_cast<float>(hc9[3] * e->pyr_scale);
        sc.dist_zero = 1;
        for (int k = 0; k < 5; ++k) { sc.d[k] = static_cast<float>(hc9[4 + k]); if (sc.d[k] != 0.0f) sc.dist_zero = 0; }
        sc.occlusion = P.occlusion_distance;
        const size_t smem = 12 * static_cast<size_t>(F) * sizeof(float);
        auto kern = (K <= 5) ? k_select_obs<5> : k_select_obs<I3D_MAX_OBS>;
        if (smem > 48 * 1024) CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        KernelTimer kt(e, "k_select_obs", 0);
        static const bool no_cull = std::getenv("I3D_NO_CULL") != nullptr;
        static const bool want_stats = std::getenv("I3D_CULL_STATS") != nullptr;
        e->cull_stats.ensure(2);
        if (want_stats) CK(cudaMemsetAsync(e->cull_stats.p, 0, 2 * sizeof(unsigned long long), st));
        CullView cull{e->tile_min.p, e->tile_max.p, no_cull ? 0 : 1, want_stats ? e->cull_stats.p : nullptr};
        pdl_launch(e, kern, blocks_for(static_cast<size_t>(n_active)), kThreads, smem, g, e->frame_view(), e->Rt.p, sc, cull, n_active, stride, e->act.p, K,
                                                                                e->obs_frame.p, e->obs_w.p);
        e->launches += 1;
        if (want_stats)
        {
            unsigned long long hs[2] = {0, 0};
            CK(cudaMemcpyAsync(hs, e->cull_stats.p, sizeof(hs), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            fprintf(stderr, "[i3d] frame culling: %llu of %llu (warp, frame) pairs visited (%.1f %%)\n", hs[0], hs[1], hs[1] ? 100.0 * hs[0] / hs[1] : 0.0);
        }
    }
    t_sel.stop();

    // ------------------------------------------------------------------ k2 build
    Timer t_build(e, "build", 2);
    e->J.ensure(static_cast<size_t>(I3D_EG_COLS) * S + 1);
    e->row_frame.ensure(S + 1); e->row_res.ensure(S + 1); e->row_wraw.ensure(S + 1); e->row_w.ensure(S + 1);
    e->ea_w.ensure(3 * static_cast<size_t>(n)); e->lap.ensure(n);
    if (apply_smem_bytes(F, K) > 48 * 1024)
    {
        CK(cudaFuncSetAttribute(k_eg_apply<APPLY_CG>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(apply_smem_bytes(F, K))));
        CK(cudaFuncSetAttribute(k_eg_apply<APPLY_MODEL>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(apply_smem_bytes(F, K))));
    }
    EgRows rows;
    rows.n_active = n_active; rows.K = K; rows.stride = stride; rows.act = e->act.p; rows.J = e->J.p; rows.row_frame = e->row_frame.p;
    rows.row_res = e->row_res.p; rows.row_wraw = e->row_wraw.p; rows.row_w = e->row_w.p;
    CamView cv{e->cam, e->pose_ctx.p, F};
    if (n_active > 0)
    {
        {
            KernelTimer kt(e, "k_eg_build", 0);
            launch_eg_rows<ROWS_BUILD>(e, g, cv, rows, e->obs_frame.p, e->obs_w.p);
        }
        const size_t smem = accum_smem_bytes(F, K);
        if (smem > 48 * 1024) CK(cudaFuncSetAttribute(k_eg_accum, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        {
            KernelTimer kt(e, "k_eg_accum");
            pdl_launch(e, k_eg_accum, blocks_for(static_cast<size_t>(n_active)), kThreads, smem, g, rows, F, e->v_bgd.p, e->v_cgd.p, e->cam_accd.p, e->site(SITE_BUILD));
        }
        pdl_launch(e, k_acc_to_float, blocks_for(std::max(U, static_cast<size_t>(lay.size()))), kThreads, 0, static_cast<int64_t>(U), lay.size(),
                   e->v_bgd.p, e->v_cgd.p, e->cam_accd.p, e->v_bg.p, e->v_cg.p, e->cam_acc.p);
        e->launches += 3;
    }
    RegView rv;
    rv.flags = e->flags.p; rv.ea_w = e->ea_w.p; rv.lap = e->lap.p;
    rv.use_er = P.use_er; rv.use_es = P.use_es; rv.use_ea = P.use_ea;
    pdl_launch(e, k_reg_build, blocks_for(static_cast<size_t>((sh.loc_end - sh.loc_begin + 3) / 4)), kThreads, 0, g, rv, sh, e->site(SITE_REG));
    {
        // active-voxel count rides along in the unused tail of SITE_BUILD
        const double na = static_cast<double>(n_active);
        CK(cudaMemcpyAsync(e->site(SITE_BUILD).out + 3, &na, sizeof(double), cudaMemcpyHostToDevice, st));
    }
    if (multi) exchange(e, e->v_bg.p, e->v_cg.p, e->cam_acc.p, lay.size(), e->red_out.p, 2 * kSiteVals, 0);   // SITE_BUILD + SITE_REG are adjacent
    // NLSSolver::normalizeCostTermWeights (nls_solver.cpp:379-394) on the device
    pdl_launch(e, k_type_weights, 1, 32, 0, e->iter_dev.p, e->site(SITE_BUILD).out, e->site(SITE_REG).out, P, n, e->type_w.p);
    if (S > 0) pdl_launch(e, k_row_weights, blocks_for(S), kThreads, 0, S, e->row_wraw.p, e->type_w.p, e->row_w.p);
    SolveVecs sv = solve_vecs(e);
    pdl_launch(e, k_finish_problem, blocks_for(static_cast<size_t>((hc + 3) / 4)), kThreads, 0, g, rv, sv, sh, hc, e->type_w.p, e->cam_acc.p, P.fix_poses, P.fix_intrinsics,
                                                                              P.fix_distortion, e->site(SITE_FINISH), e->cam);
    allreduce_scalars(e, e->site(SITE_FINISH).out, 3, -1, 0);
    pdl_launch(e, k_iter_finish, 1, 32, 0, e->iter_dev.p, e->site(SITE_FINISH).out, P);
    e->launches += 5;
    t_build.stop();
    e->have_iter = true;
    if (P.build_only)
    {
        IterDev hb{};
        CK(cudaMemcpyAsync(&hb, e->iter_dev.p, sizeof(hb), cudaMemcpyDeviceToHost, st));
        sync();
        CK(cudaGetLastError());
        info = hb.info;
        t_total.stop();
        return 0;
    }

    // ------------------------------------------------------------------ LM loop (TrustRegionMinimizer + LevenbergMarquardtStrategy)
    Timer t_solve(e, "solve", 3);
    const float dmin = static_cast<float>(P.min_lm_diagonal), dmax = static_cast<float>(std::min(P.max_lm_diagonal, 3.0e38));
    // voxel unknowns: 4 per thread (16 B accesses) in the single-GPU identity layout, 1 per thread through the held list when sharded
    // voxel unknowns of the held hull: 4 per thread (16 B accesses); the first F + 2 threads take one camera block each
    const unsigned upd_blocks = blocks_for(static_cast<size_t>((sh.held_voxel_unknowns() + 3) / 4 + F + 2));
    auto launch_update = [&](bool init, int refresh) {
        if (init) pdl_launch(e, (k_cg_update<true, 4>), upd_blocks, kThreads, 0, sv, sh, e->minv.p, dmin, dmax, e->ctl.p, refresh, e->site(SITE_UPDATE));
        else pdl_launch(e, (k_cg_update<false, 4>), upd_blocks, kThreads, 0, sv, sh, e->minv.p, dmin, dmax, e->ctl.p, refresh, e->site(SITE_UPDATE));
        e->launches += 1;
    };
    const unsigned vec_blocks = blocks_for(static_cast<size_t>(hc));
    const int max_it = P.forced_cg_iterations > 0 ? P.forced_cg_iterations : P.max_linear_solver_iterations;
    int enq = 0;                 // PCG iterations enqueued in the current trial
    auto enqueue_pcg = [&](int count) {
        for (int bidx = 0; bidx < count && enq < max_it; ++bidx)
        {
            ++enq;
            const bool refresh = (enq % P.residual_reset_period == 0);
            {
                KernelTimer kt(e, "k_cg_dir");
                pdl_launch(e, k_cg_dir4, blocks_for(static_cast<size_t>((hc + 3) / 4)), kThreads, 0, sv, sh, hc, e->ctl.p);
                e->launches += 1;
            }
            launch_operator(e, g, rv, rows, sv, sh, sv.p, dmin, dmax, 1, enq == 1);
            if (refresh)
            {
                // exact residual: x += alpha p ; r = b - A x   (needs the operator's qg consumed first: do the plain update
                // of x only, then apply the operator to x)
                pdl_launch(e, k_x_update, vec_blocks, kThreads, 0, sv, sh, hc, e->ctl.p);
                // discard A p: k_cg_update(refresh) below consumes A x, so clear qg by a dry consume
                CK(cudaMemsetAsync(e->v_qg.p, 0, U * sizeof(float), st));
                pdl_launch(e, k_scale_vec, vec_blocks, kThreads, 0, sv, sh, hc, sv.x, 1.0f, sv.ps, e->ctl.p, 1);
                e->launches += 2;
                launch_operator(e, g, rv, rows, sv, sh, sv.x, dmin, dmax, 0);
                launch_update(false, 1);
            }
            else
            {
                KernelTimer kt(e, "k_cg_update");
                launch_update(false, 0);
            }
            if (multi) allreduce_scalars(e, e->site(SITE_UPDATE).out, 3, EPI_UPDATE, 1);
        }
    };
    // candidate point + candidate cost + the trust-region decision, all stream-ordered behind the PCG.  The model cost change comes
    // from the PCG's own scalars (k_lm_decide): no extra pass over the Jacobian.
    auto enqueue_decision = [&]() {
        Timer t_cand(e, "candidate", 5);
        CK(cudaMemsetAsync(e->red_out.p + SITE_CAND * kSiteVals, 0, 3 * kSiteVals * sizeof(double), st));
        pdl_launch(e, k_candidate, vec_blocks, kThreads, 0, g, sv, sh, hc, 0, e->cam, e->c_sdf, e->c_alb, e->c_cam, e->v_delta.p, e->ctl.p, e->site(SITE_CAND));
        GridView gc = e->grid_view(e->c_sdf, e->c_alb);
        pdl_launch(e, k_frame_pose, blocks_for(F, 64), 64, 0, F, e->c_cam, e->pose_ctx_c.p);
        CamView cvc{e->c_cam, e->pose_ctx_c.p, F};
        if (n_active > 0)
        {
            KernelTimer kt(e, "k_eg_cost", 0);
            launch_eg_rows<ROWS_COST>(e, gc, cvc, rows, nullptr, nullptr);
        }
        pdl_launch(e, k_reg_cost, blocks_for(static_cast<size_t>(own)), kThreads, 0, gc, rv, sh, e->c_sdf, e->c_alb, e->site(SITE_REG_COST));
        if (multi) allreduce_scalars(e, e->red_out.p + SITE_CAND * kSiteVals, 3 * kSiteVals, -1, 0);   // SITE_CAND, SITE_EG_COST, SITE_REG_COST are adjacent
        pdl_launch(e, k_lm_decide, 1, 32, 0, e->iter_dev.p, e->ctl.p, e->fail_flag.p, e->site(SITE_CAND).out, e->site(SITE_EG_COST).out,
                                      e->site(SITE_REG_COST).out, e->type_w.p, P);
        e->launches += 5;
    };
    IterDev h{};
    for (int it = 1; it <= P.lm_steps; ++it)
    {
        Timer t_pcg(e, "pcg", 4);
        pdl_launch(e, k_lm_begin, 1, 32, 0, e->iter_dev.p, e->ctl.p, e->fail_flag.p, P);
        pdl_launch(e, k_cam_precond, blocks_for(static_cast<size_t>(F) + 2, 64), 64, 0, sv, e->cam_acc.p, e->type_w.p, e->ctl.p, dmin, dmax, e->minv.p, e->fail_flag.p);
        e->launches += 2;
        launch_update(true, 0);
        if (multi) allreduce_scalars(e, e->site(SITE_UPDATE).out, 3, EPI_UPDATE_INIT, 0);
        enq = 0;
        // Kernels of iterations enqueued past convergence are no-ops but still cost a grid launch each, and every extra round
        // costs a host round trip plus a wasted decision phase: enqueue as many iterations as the larger of the previous two solves
        // needed (the counts alternate, e.g. 5, 4, 5, ...), then the decision; k_lm_decide reports an unfinished solve and the host
        // adds iterations two at a time.
        enqueue_pcg(P.forced_cg_iterations > 0 ? P.forced_cg_iterations : std::max(e->last_cg_iterations, e->prev_cg_iterations));
        t_pcg.stop();
        while (true)
        {
            enqueue_decision();
            CK(cudaMemcpyAsync(&h, e->iter_dev.p, sizeof(h), cudaMemcpyDeviceToHost, st));
            sync();
            CK(cudaGetLastError());
            if (!h.pcg_unfinished || h.state != LM_RUNNING) break;
            Timer t_more(e, "pcg", 4);
            enqueue_pcg(2);
        }
        if (h.info.lm_iterations >= 1)
        {
            e->prev_cg_iterations = e->last_cg_iterations;
            e->last_cg_iterations = std::max(1, h.info.cg_iterations[std::min(h.info.lm_iterations - 1, I3D_MAX_LM_STEPS - 1)]);
        }
        if (h.state != LM_RUNNING) break;
    }
    info = h.info;
    if (h.precond_fail) e->error = "camera preconditioner block not SPD";
    if (h.state == LM_ACCEPTED)
    {
        if (multi)
        {
            // every rank needs the complete new state: sum the owned parts of the step, rebuild the candidate for all unknowns
            pdl_launch(e, k_mask_owned, blocks_for(U), kThreads, 0, sv, sh, e->v_delta.p);
            NK(g_nccl.AllReduce(e->v_delta.p, e->v_delta.p, U, NCCL_FLOAT32, NCCL_SUM, e->comm, st));
            pdl_launch(e, k_candidate, blocks_for(U), kThreads, 0, g, sv, sh, static_cast<int64_t>(U), 1, e->cam, e->c_sdf, e->c_alb, e->c_cam, e->v_delta.p, e->ctl.p,
                                                           e->site(SITE_CAND));
            sync();
            e->launches += 2;
        }
        std::swap(e->sdf, e->c_sdf); std::swap(e->alb, e->c_alb); std::swap(e->cam, e->c_cam);
    }
    t_solve.stop();
    t_total.stop();
    return 0;
}

// builds the held / shared bookkeeping of this rank's shard (static per grid + shard)
int setup_shard(I3DEngine* e)
{
    const int64_t n = e->n;
    const int64_t n2 = 2 * n;
    cudaStream_t st = e->stream;
    Shard sh0;
    sh0.own_begin = e->shard_begin; sh0.own_end = e->shard_end; sh0.hv0 = 0; sh0.hv1 = n; sh0.cam_owner = (e->rank == 0); sh0.defer = 1; sh0.loc_begin = 0; sh0.loc_end = n;
    Dev<uint8_t> touch, count;
    touch.ensure(n2); count.ensure(n2);
    CK(cudaMemsetAsync(touch.p, 0, n2, st));
    GridView g = e->grid_view(e->sdf, e->alb);
    const int64_t own = e->shard_end - e->shard_begin;
    if (own > 0) k_touch<<<blocks_for(static_cast<size_t>(own)), kThreads, 0, st>>>(g, sh0, touch.p);
    CK(cudaMemcpyAsync(count.p, touch.p, n2, cudaMemcpyDeviceToDevice, st));
    NK(g_nccl.AllReduce(count.p, count.p, static_cast<size_t>(n2), NCCL_UINT8, NCCL_SUM, e->comm, st));
    e->held.ensure(n2); e->held_mask.ensure(n2);
    k_share_flags<<<blocks_for(static_cast<size_t>(n2)), kThreads, 0, st>>>(n2, touch.p, count.p, e->held.p);
    CK(cudaMemcpyAsync(e->held_mask.p, touch.p, n2, cudaMemcpyDeviceToDevice, st));
    // compaction: shared list (bit1) and held list (bit0)
    const int nscan = static_cast<int>((n2 + kScanChunk - 1) / kScanChunk);
    e->scan_counts.ensure(nscan); e->scan_total.ensure(1);
    e->slist.ensure(n2);
    int32_t tot = 0;
    k_scan_count<<<nscan, kThreads, 0, st>>>(n2, e->held.p, 2, e->scan_counts.p);
    k_scan_blocks<<<1, 1024, 0, st>>>(nscan, e->scan_counts.p, e->scan_total.p);
    k_scan_scatter<<<nscan, kThreads, 0, st>>>(n2, e->held.p, 2, e->scan_counts.p, e->slist.p);
    CK(cudaMemcpyAsync(&tot, e->scan_total.p, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    e->n_shared = tot;
    // index range of everything this rank reads per iteration: flags / E_r / E_a data of the held voxels' rings need the state of
    // own + 4 stencil rings (held = 1, their 6-ring = 2, the +x/+y/+z pair partners = 3, the forward-difference normal = 4)
    {
        int64_t lo = e->shard_begin, hi = e->shard_end;
        Dev<int> mm; mm.ensure(2);
        for (int round = 0; round < 4 && hi > lo; ++round)
        {
            const int init[2] = {INT_MAX, -1};
            CK(cudaMemcpyAsync(mm.p, init, sizeof(init), cudaMemcpyHostToDevice, st));
            k_range_extend<<<blocks_for(static_cast<size_t>(hi - lo)), kThreads, 0, st>>>(g, lo, hi, mm.p);
            int out[2];
            CK(cudaMemcpyAsync(out, mm.p, sizeof(out), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            lo = std::min<int64_t>(lo, out[0]); hi = std::max<int64_t>(hi, static_cast<int64_t>(out[1]) + 1);
            if (round == 0)
            {
                // round 1 = own voxels + their stencil = the voxels whose unknowns this rank holds: their index hull, widened to
                // multiples of 4 so that the per-unknown kernels can use 16 B accesses
                e->hv0 = lo & ~static_cast<int64_t>(3);
                e->hv1 = std::min<int64_t>(n, (hi + 3) & ~static_cast<int64_t>(3));
            }
        }
        if (e->shard_end <= e->shard_begin) { e->hv0 = 0; e->hv1 = 0; }
        e->loc_begin = std::min(lo, e->hv0); e->loc_end = std::max(hi, e->hv1);
    }
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    e->shard_ready = true;
    return 0;
}

} // namespace

// =================================================================================================
// C-ABI
// =================================================================================================
extern "C" {

int i3d_abi_version(void) { return I3D_ABI_VERSION; }
uint64_t i3d_sizeof_params(void) { return sizeof(I3DParams); }
uint64_t i3d_sizeof_iter_info(void) { return sizeof(I3DIterInfo); }

void i3d_default_params(I3DParams* p)
{
    std::memset(p, 0, sizeof(*p));
    p->lambda[0] = 0.2; p->lambda[1] = 80.0; p->lambda[2] = 120.0; p->lambda[3] = 0.1;
    p->use_er = p->use_es = p->use_ea = 1;
    p->occlusion_distance = 0.02f; p->num_observations = 5; p->lm_steps = 50;
    p->initial_trust_region_radius = 1e4; p->max_trust_region_radius = 1e16; p->min_trust_region_radius = 1e-32;
    p->min_relative_decrease = 1e-3; p->min_lm_diagonal = 1e-6; p->max_lm_diagonal = 1e32; p->eta = 0.1;
    p->function_tolerance = 1e-6; p->gradient_tolerance = 1e-10; p->parameter_tolerance = 1e-8;
    p->max_linear_solver_iterations = 500; p->min_linear_solver_iterations = 0; p->residual_reset_period = 10;
    p->max_consecutive_invalid_steps = 5;
}

int i3d_engine_create(int device, I3DEngine** out)
{
    *out = nullptr;
    int count = 0;
    cudaError_t err = cudaGetDeviceCount(&count);
    if (err != cudaSuccess || count <= 0) return fail(nullptr, "i3d_engine_create: no CUDA device available (%s); this engine has no CPU fallback", cudaGetErrorString(err));
    if (device < 0 || device >= count) return fail(nullptr, "i3d_engine_create: device %d out of range (%d devices)", device, count);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, "i3d_engine_create: cannot query device %d", device);
    // arch-specific sm_90a code runs on compute capability 9.0 only
    if (prop.major != 9 || prop.minor != 0) return fail(nullptr, "i3d_engine_create: device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
    I3DEngine* e = new I3DEngine();
    e->device = device;
    const int rc = guarded(e, [&]() {
        CK(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
        for (auto& ev : e->ev) CK(cudaEventCreate(&ev));
        e->ev_pool.resize(4096);
        for (auto& ev : e->ev_pool) CK(cudaEventCreate(&ev));
        return 0;
    });
    if (rc != 0) { g_create_error = e->error; delete e; return rc; }
    *out = e;
    return 0;
}

void i3d_engine_destroy(I3DEngine* e)
{
    if (!e) return;
    cudaSetDevice(e->device);
    cudaStreamSynchronize(e->stream);
    for (size_t r = 0; r < e->peer_base.size(); ++r)
        if (static_cast<int>(r) != e->rank && e->peer_base[r]) cudaIpcCloseMemHandle(e->peer_base[r]);
    if (e->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(e->comm);
    for (auto& ev : e->ev) cudaEventDestroy(ev);
    for (auto& ev : e->ev_pool) cudaEventDestroy(ev);
    cudaStreamDestroy(e->stream);
    delete e;
}

const char* i3d_last_error(const I3DEngine* e) { return e ? e->error.c_str() : g_create_error.c_str(); }

int i3d_upload_grid(I3DEngine* e, int64_t n, const int32_t* xyz, const double* sdf0, const double* sdf_refined, const double* albedo,
                    const float* weight, const uint8_t* rgb, float voxel_size)
{
    if (!e) return 1;
    if (n <= 0 || n > (1ll << 30)) return fail(e, "i3d_upload_grid: bad voxel count %lld", static_cast<long long>(n));
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        e->n = n; e->voxel_size = voxel_size; e->truncation = voxel_size * 5.0f; e->have_sh = false; e->have_iter = false; e->shard_ready = false; e->sv_S = 0; e->sv_x = nullptr;
        e->x.ensure(n); e->y.ensure(n); e->z.ensure(n); e->nbr.ensure(static_cast<size_t>(NB_COUNT) * n);
        e->sdf0.ensure(n); e->sdfA.ensure(n); e->sdfB.ensure(n); e->albA.ensure(n); e->albB.ensure(n); e->weight.ensure(n); e->rgb.ensure(n);
        e->sdf = e->sdfA.p; e->c_sdf = e->sdfB.p; e->alb = e->albA.p; e->c_alb = e->albB.p;
        e->up_xyz.ensure(3 * static_cast<size_t>(n)); e->up_rgb.ensure(3 * static_cast<size_t>(n));
        CK(cudaMemcpyAsync(e->up_xyz.p, xyz, 3 * n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(e->up_rgb.p, rgb, 3 * n, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(e->sdf0.p, sdf0, n * sizeof(double), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(e->sdf, sdf_refined, n * sizeof(double), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(e->alb, albedo, n * sizeof(double), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(e->weight.p, weight, n * sizeof(float), cudaMemcpyHostToDevice, st));
        k_deinterleave_xyz<<<blocks_for(n), kThreads, 0, st>>>(n, e->up_xyz.p, e->x.p, e->y.p, e->z.p, e->up_rgb.p, e->rgb.p);
        const int hdup = rebuild_topology(e);
        if (hdup) return fail(e, "i3d_upload_grid: duplicate voxel coordinates");
        return 0;
    });
}

int i3d_upload_voxel_params(I3DEngine* e, const double* sdf_refined, const double* albedo)
{
    if (!e || e->n <= 0) return fail(e, "i3d_upload_voxel_params: no grid");
    return guarded(e, [&]() {
        if (sdf_refined) CK(cudaMemcpyAsync(e->sdf, sdf_refined, e->n * sizeof(double), cudaMemcpyHostToDevice, e->stream));
        if (albedo) CK(cudaMemcpyAsync(e->alb, albedo, e->n * sizeof(double), cudaMemcpyHostToDevice, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        return 0;
    });
}

int i3d_upload_frames(I3DEngine* e, int32_t F, int32_t W, int32_t H, const float* lum, const float* depth, double pyr_scale)
{
    if (!e) return 1;
    if (F <= 0 || W <= 0 || H <= 0) return fail(e, "i3d_upload_frames: bad dimensions");
    return guarded(e, [&]() {
        const size_t cnt = static_cast<size_t>(F) * W * H;
        if (F != e->F) { e->have_cam = false; e->have_iter = false; }     // the unknown space of the last iteration no longer matches
        if (F != e->F || W != e->W || H != e->H) e->have_color = false;
        e->F = F; e->W = W; e->H = H; e->pyr_scale = pyr_scale;
        e->lum.ensure(cnt); e->depth.ensure(cnt);
        // The live camera state may sit in camB (every accepted LM step swaps cam / c_cam): a re-upload of the frames of another
        // pyramid level with the SAME frame count must not touch it.  Only a new frame count (camera invalidated above) or a first
        // allocation resets the pair.
        if (!e->have_cam || e->cam == nullptr)
        {
            e->camA.ensure(6 * static_cast<size_t>(F) + 9); e->camB.ensure(6 * static_cast<size_t>(F) + 9);
            e->cam = e->camA.p; e->c_cam = e->camB.p;
        }
        CK(cudaMemcpyAsync(e->lum.p, lum, cnt * sizeof(float), cudaMemcpyHostToDevice, e->stream));
        CK(cudaMemcpyAsync(e->depth.p, depth, cnt * sizeof(float), cudaMemcpyHostToDevice, e->stream));
        {
            const int TW = (W + kCullTile - 1) / kCullTile, TH = (H + kCullTile - 1) / kCullTile;
            const size_t nt = static_cast<size_t>(F) * TW * TH;
            e->tile_min.ensure(nt); e->tile_max.ensure(nt);
            k_depth_tiles<<<static_cast<unsigned>(nt), 256, 0, e->stream>>>(F, W, H, e->depth.p, e->tile_min.p, e->tile_max.p);
        }
        CK(cudaStreamSynchronize(e->stream));
        CK(cudaGetLastError());
        return 0;
    });
}

int i3d_set_camera(I3DEngine* e, const double* poses, const double* intrinsics, const double* distortion)
{
    if (!e || e->F <= 0) return fail(e, "i3d_set_camera: upload frames first");
    return guarded(e, [&]() {
        const size_t F = static_cast<size_t>(e->F);
        CK(cudaMemcpyAsync(e->cam, poses, 6 * F * sizeof(double), cudaMemcpyHostToDevice, e->stream));
        CK(cudaMemcpyAsync(e->cam + 6 * F, intrinsics, 4 * sizeof(double), cudaMemcpyHostToDevice, e->stream));
        CK(cudaMemcpyAsync(e->cam + 6 * F + 4, distortion, 5 * sizeof(double), cudaMemcpyHostToDevice, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        e->have_cam = true;
        return 0;
    });
}

int i3d_set_sh(I3DEngine* e, const double* sh9n)
{
    if (!e || e->n <= 0) return fail(e, "i3d_set_sh: upload the grid first");
    return guarded(e, [&]() {
        const size_t cnt = 9 * static_cast<size_t>(e->n);
        e->up_sh.ensure(cnt);
        e->sh.ensure(cnt);
        CK(cudaMemcpyAsync(e->up_sh.p, sh9n, cnt * sizeof(double), cudaMemcpyHostToDevice, e->stream));
        k_transpose_sh<<<blocks_for(cnt), kThreads, 0, e->stream>>>(e->n, e->up_sh.p, e->sh.p);
        e->sh_has.ensure(static_cast<size_t>(e->n));
        CK(cudaMemsetAsync(e->sh_has.p, 1, static_cast<size_t>(e->n), e->stream));
        CK(cudaStreamSynchronize(e->stream));
        CK(cudaGetLastError());
        e->have_sh = true;
        return 0;
    });
}

int i3d_gn_iteration(I3DEngine* e, const I3DParams* params, I3DIterInfo* info)
{
    if (!e || !params || !info) return 1;
    return guarded(e, [&]() {
        const int rc = gn_iteration_impl(e, *params, *info);
        collect_kernel_times(e);
        // the reference's three phase timers (NLSSolver::ProblemInfo::time_add/time_build, SolverInfo::time_solve)
        info->time_add = (e->phases["select"].ms + e->phases["build"].ms) * 1e-3;
        info->time_build = 0.0;
        info->time_solve = e->phases["solve"].ms * 1e-3;
        return rc;
    });
}

int i3d_download_state(I3DEngine* e, double* sdf_refined, double* albedo, double* poses, double* intrinsics, double* distortion)
{
    if (!e || e->n <= 0) return fail(e, "i3d_download_state: no grid");
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t F = static_cast<size_t>(e->F);
        if (sdf_refined) CK(cudaMemcpyAsync(sdf_refined, e->sdf, e->n * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (albedo) CK(cudaMemcpyAsync(albedo, e->alb, e->n * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (poses && F) CK(cudaMemcpyAsync(poses, e->cam, 6 * F * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (intrinsics && F) CK(cudaMemcpyAsync(intrinsics, e->cam + 6 * F, 4 * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (distortion && F) CK(cudaMemcpyAsync(distortion, e->cam + 6 * F + 4, 5 * sizeof(double), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    });
}

// ---- SVSH lighting ----------------------------------------------------------------------------
uint64_t i3d_sizeof_lighting_params(void) { return sizeof(I3DLightingParams); }
uint64_t i3d_sizeof_lighting_info(void) { return sizeof(I3DLightingInfo); }

void i3d_default_lighting_params(I3DLightingParams* p)
{
    std::memset(p, 0, sizeof(*p));
    p->subvolume_size = 0.2f; p->weighted = 1; p->lambda_reg = 10.0; p->thres_shell = 0.0;
    p->max_iterations = 50; p->max_linear_solver_iterations = 500; p->min_linear_solver_iterations = 0; p->residual_reset_period = 10;
    p->max_consecutive_invalid_steps = 5;
    p->initial_trust_region_radius = 1e4; p->max_trust_region_radius = 1e16; p->min_trust_region_radius = 1e-32;
    p->min_relative_decrease = 1e-3; p->min_lm_diagonal = 1e-6; p->max_lm_diagonal = 1e32; p->eta = 0.1;
    p->function_tolerance = 1e-6; p->gradient_tolerance = 1e-10; p->parameter_tolerance = 1e-8;
}

int i3d_estimate_lighting(I3DEngine* e, const I3DLightingParams* params, I3DLightingInfo* info)
{
    if (!e || !params || !info) return 1;
    std::memset(info, 0, sizeof(*info));
    info->termination = 2;
    if (e->n <= 0 && e->x.p != nullptr) return 0;      // grid emptied by the pruning: LightingSVSH::estimate() returns false (no subvolumes)
    if (e->n <= 0) return fail(e, "i3d_estimate_lighting: upload the grid first");
    const I3DLightingParams P = *params;
    if (!(P.thres_shell > 0.0)) return 0;        // LightingSVSH::estimate returns false (lighting_svsh.cpp:170)
    // the reference registers one parameter block twice in a residual block for a single volume (size <= 0): ceres aborts
    if (!(P.subvolume_size > 0.0f)) return fail(e, "i3d_estimate_lighting: subvolume_size must be > 0");
    if (P.residual_reset_period <= 0 || P.max_iterations < 0) return fail(e, "i3d_estimate_lighting: bad solver options");
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const int64_t n = e->n;
        e->timed.clear(); e->ev_used = 0;
        for (const char* nm : {"light_subvolumes", "light_accumulate", "light_solve", "light_interpolate"}) e->phases.erase(nm);
        const GridView g = e->grid_view(e->sdf, e->alb);
        SubvolGrid sg;
        sg.inv_size = 1.0f / P.subvolume_size;
        // ---- Subvolumes::compute ----
        e->sv_scalars.ensure(8);
        {
            Timer t(e, "light_subvolumes", 0);
            const int init[7] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN, 0};
            CK(cudaMemcpyAsync(e->sv_scalars.p, init, sizeof(init), cudaMemcpyHostToDevice, st));
            k_svsh_bounds<<<blocks_for(n), kThreads, 0, st>>>(n, e->x.p, e->y.p, e->z.p, e->voxel_size, sg.inv_size, e->sv_scalars.p);
            int bounds[6];
            CK(cudaMemcpyAsync(bounds, e->sv_scalars.p, sizeof(bounds), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            int64_t cells = 1;
            for (int d = 0; d < 3; ++d)
            {
                sg.lo[d] = bounds[d];
                const int64_t ext = static_cast<int64_t>(bounds[3 + d]) - bounds[d] + 1;
                if (ext <= 0 || ext > (1 << 24)) return fail(e, "i3d_estimate_lighting: bad subvolume bounds");
                sg.dim[d] = static_cast<int>(ext);
                cells *= ext;
                if (cells > (1ll << 24)) return fail(e, "i3d_estimate_lighting: subvolume bounding box too large (%lld cells); increase subvolume_size", static_cast<long long>(cells));
            }
            e->sv_table.ensure(static_cast<size_t>(cells));
            sg.table = e->sv_table.p;
            CK(cudaMemsetAsync(e->sv_table.p, 0, static_cast<size_t>(cells) * sizeof(int32_t), st));
            k_svsh_mark<<<blocks_for(n), kThreads, 0, st>>>(n, e->x.p, e->y.p, e->z.p, e->voxel_size, sg, e->sv_table.p);
            k_svsh_number<<<1, kLightSolveThreads, 0, st>>>(cells, e->sv_table.p, e->sv_scalars.p + 6);
            int S = 0;
            CK(cudaMemcpyAsync(&S, e->sv_scalars.p + 6, sizeof(int), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            CK(cudaGetLastError());
            if (S <= 0) return fail(e, "i3d_estimate_lighting: no subvolumes");
            e->sv_S = S;
            e->sv_index.ensure(3 * static_cast<size_t>(S)); e->sv_nbr.ensure(6 * static_cast<size_t>(S)); e->sv_deg.ensure(static_cast<size_t>(S));
            k_svsh_indices<<<blocks_for(static_cast<size_t>(cells)), kThreads, 0, st>>>(sg, e->sv_index.p, e->sv_nbr.p, S);
        }
        const int S = e->sv_S;
        const size_t M = 9 * static_cast<size_t>(S);
        // ---- data rows -> per-subvolume normal equations ----
        e->sv_acc.ensure(static_cast<size_t>(S) * kLightAcc);
        {
            Timer t(e, "light_accumulate", 0);
            CK(cudaMemsetAsync(e->sv_acc.p, 0, static_cast<size_t>(S) * kLightAcc * sizeof(double), st));
            k_svsh_accumulate<<<blocks_for(n), kThreads, 0, st>>>(g, sg, P.thres_shell, P.weighted != 0, e->sv_acc.p);
        }
        // ---- ceres::Solve on the reduced system, one launch ----
        e->sv_work.ensure(162 * static_cast<size_t>(S) + 14 * M);
        e->sv_info.ensure(1);
        LightSolveWork W;
        {
            double* w = e->sv_work.p;
            W.S = S; W.acc = e->sv_acc.p; W.nbr = e->sv_nbr.p; W.deg = e->sv_deg.p; W.info = e->sv_info.p;
            W.H = w; w += 81 * static_cast<size_t>(S);
            W.Minv = w; w += 81 * static_cast<size_t>(S);
            double** vecs[] = {&W.g, &W.scale, &W.diag, &W.D2, &W.gU, &W.x, &W.b, &W.xs, &W.r, &W.z, &W.p, &W.q, &W.t, &W.w};
            for (double** v : vecs) { *v = w; w += M; }
            e->sv_x = W.x;
        }
        {
            Timer t(e, "light_solve", 0);
            CK(cudaMemsetAsync(e->sv_info.p, 0, sizeof(I3DLightingInfo), st));
            k_svsh_solve<<<1, kLightSolveThreads, 0, st>>>(W, P);
        }
        CK(cudaMemcpyAsync(info, e->sv_info.p, sizeof(I3DLightingInfo), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        CK(cudaGetLastError());
        if (info->usable)
        {
            // ---- computeVoxelShCoeffs ----
            e->sh.ensure(9 * static_cast<size_t>(n)); e->sh_has.ensure(static_cast<size_t>(n));
            Timer t(e, "light_interpolate", 0);
            k_svsh_interpolate<<<blocks_for(n), kThreads, 0, st>>>(g, sg, P.thres_shell, e->sv_x, e->sh.p, e->sh_has.p);
            t.stop();
            e->have_sh = true;
        }
        collect_kernel_times(e);
        CK(cudaGetLastError());
        info->time_accumulate = (e->phases["light_subvolumes"].ms + e->phases["light_accumulate"].ms) * 1e-3;
        info->time_solve = e->phases["light_solve"].ms * 1e-3;
        info->time_interpolate = e->phases["light_interpolate"].ms * 1e-3;
        return 0;
    });
}

int64_t i3d_lighting_num_subvolumes(const I3DEngine* e) { return e ? e->sv_S : 0; }

int i3d_download_lighting(I3DEngine* e, int32_t* subvolume_index3, double* sh9)
{
    if (!e || e->sv_S <= 0 || !e->sv_x) return fail(e, "i3d_download_lighting: no lighting estimate");
    return guarded(e, [&]() {
        const size_t S = static_cast<size_t>(e->sv_S);
        if (subvolume_index3) CK(cudaMemcpyAsync(subvolume_index3, e->sv_index.p, 3 * S * sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
        if (sh9) CK(cudaMemcpyAsync(sh9, e->sv_x, 9 * S * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        return 0;
    });
}

int i3d_download_voxel_sh(I3DEngine* e, double* sh9n, uint8_t* has_sh)
{
    if (!e || e->n <= 0 || !e->have_sh) return fail(e, "i3d_download_voxel_sh: no per-voxel SH on the device");
    return guarded(e, [&]() {
        const size_t cnt = 9 * static_cast<size_t>(e->n);
        if (sh9n)
        {
            e->up_sh.ensure(cnt);
            k_untranspose_sh<<<blocks_for(cnt), kThreads, 0, e->stream>>>(e->n, e->sh.p, e->up_sh.p);
            CK(cudaMemcpyAsync(sh9n, e->up_sh.p, cnt * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
        }
        if (has_sh) CK(cudaMemcpyAsync(has_sh, e->sh_has.p, static_cast<size_t>(e->n), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        CK(cudaGetLastError());
        return 0;
    });
}

// ---- voxel recolouring ------------------------------------------------------------------------
int i3d_upload_color_frames(I3DEngine* e, const uint8_t* bgr)
{
    if (!e || !bgr) return 1;
    if (e->F <= 0) return fail(e, "i3d_upload_color_frames: upload the depth / luminance frames first");
    return guarded(e, [&]() {
        const size_t cnt = static_cast<size_t>(e->F) * e->W * e->H * 3;
        e->color.ensure(cnt);
        CK(cudaMemcpyAsync(e->color.p, bgr, cnt, cudaMemcpyHostToDevice, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        e->have_color = true;
        return 0;
    });
}

int i3d_recompute_colors(I3DEngine* e, const float* pose_world_to_cam, float max_occlusion_distance, int32_t max_num_observations, int64_t* num_recolored,
                         int64_t* num_observations)
{
    if (!e) return 1;
    if (e->n <= 0 || e->F <= 0 || !e->have_cam) return fail(e, "i3d_recompute_colors: grid, frames and camera must be uploaded first");
    if (!e->have_color) return fail(e, "i3d_recompute_colors: no colour frames (i3d_upload_color_frames)");
    if (max_num_observations < 0 || max_num_observations > I3D_MAX_OBS) return fail(e, "i3d_recompute_colors: max_num_observations must be in [0, %d]", I3D_MAX_OBS);
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const int F = e->F, K = max_num_observations;
        e->timed.clear(); e->ev_used = 0; e->phases.erase("recolor");
        double hc9[9];
        CK(cudaMemcpyAsync(hc9, e->cam + 6 * static_cast<size_t>(F), 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        e->Rt.ensure(12 * static_cast<size_t>(F));
        e->recolor_counts.ensure(2);
        CK(cudaMemsetAsync(e->recolor_counts.p, 0, 2 * sizeof(unsigned long long), st));
        {
            Timer t(e, "recolor", 0);
            if (pose_world_to_cam) CK(cudaMemcpyAsync(e->Rt.p, pose_world_to_cam, 12 * static_cast<size_t>(F) * sizeof(float), cudaMemcpyHostToDevice, st));
            else k_pose_mats<<<blocks_for(F, 64), 64, 0, st>>>(F, e->cam, e->Rt.p);
            SelectCam sc;
            sc.fx = static_cast<float>(hc9[0] * e->pyr_scale); sc.fy = static_cast<float>(hc9[1] * e->pyr_scale);
            sc.cx = static_cast<float>(hc9[2] * e->pyr_scale); sc.cy = static_cast<float>(hc9[3] * e->pyr_scale);
            sc.dist_zero = 1;
            for (int k = 0; k < 5; ++k) { sc.d[k] = static_cast<float>(hc9[4 + k]); if (sc.d[k] != 0.0f) sc.dist_zero = 0; }
            sc.occlusion = max_occlusion_distance;
            const size_t smem = 12 * static_cast<size_t>(F) * sizeof(float);
            auto kern = (K <= 5) ? k_recolor<5> : k_recolor<I3D_MAX_OBS>;
            if (smem > 48 * 1024) CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
            static const bool no_cull = std::getenv("I3D_NO_CULL") != nullptr;
            CullView cull{e->tile_min.p, e->tile_max.p, no_cull ? 0 : 1, nullptr};
            kern<<<blocks_for(static_cast<size_t>(e->n)), kThreads, smem, st>>>(e->grid_view(e->sdf, e->alb), e->frame_view(), e->color.p, e->Rt.p, sc, cull, K,
                                                                               e->rgb.p, e->recolor_counts.p);
        }
        unsigned long long hcnt[2] = {0, 0};
        CK(cudaMemcpyAsync(hcnt, e->recolor_counts.p, sizeof(hcnt), cudaMemcpyDeviceToHost, st));
        collect_kernel_times(e);
        CK(cudaGetLastError());
        if (num_recolored) *num_recolored = static_cast<int64_t>(hcnt[0]);
        if (num_observations) *num_observations = static_cast<int64_t>(hcnt[1]);
        return 0;
    });
}

int i3d_download_colors(I3DEngine* e, uint8_t* rgb3n)
{
    if (!e || e->n <= 0 || !rgb3n) return fail(e, "i3d_download_colors: no grid");
    return guarded(e, [&]() {
        e->up_rgb.ensure(3 * static_cast<size_t>(e->n));
        k_interleave_rgb<<<blocks_for(e->n), kThreads, 0, e->stream>>>(e->n, e->rgb.p, e->up_rgb.p);
        CK(cudaMemcpyAsync(rgb3n, e->up_rgb.p, 3 * static_cast<size_t>(e->n), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        CK(cudaGetLastError());
        return 0;
    });
}

// ---- grid-level transitions -------------------------------------------------------------------
int64_t i3d_num_voxels(const I3DEngine* e) { return e ? e->n : 0; }

int i3d_clear_voxels_outside_thin_shell(I3DEngine* e, double thres_shell, int64_t* num_voxels_out)
{
    if (!e || e->n <= 0) return fail(e, "i3d_clear_voxels_outside_thin_shell: upload the grid first");
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const int64_t n = e->n;
        e->timed.clear(); e->ev_used = 0; e->phases.erase("prune");
        Dev<int32_t>&nx = e->sp_x, &ny = e->sp_y, &nz = e->sp_z; Dev<double>&nsdf0 = e->sp_sdf0, &nsdf = e->sp_sdf, &nalb = e->sp_alb; Dev<float>& nw = e->sp_w; Dev<uchar4>& nrgb = e->sp_rgb;
        int m = 0;
        {
            Timer t(e, "prune", 0);
            const GridView g = e->grid_view(e->sdf, e->alb);
            e->flags.ensure(static_cast<size_t>(n));
            CK(cudaMemsetAsync(e->flags.p, 0, static_cast<size_t>(n), st));
            k_shell_keep<<<blocks_for(n), kThreads, 0, st>>>(g, thres_shell, e->flags.p);
            k_shell_crossing<<<blocks_for(n), kThreads, 0, st>>>(g, e->up_keys.p, e->up_vals.p, e->hash_cap - 1, e->flags.p);
            const int nscan = static_cast<int>((n + kScanChunk - 1) / kScanChunk);
            e->scan_counts.ensure(static_cast<size_t>(nscan) + 1); e->scan_total.ensure(1); e->act.ensure(static_cast<size_t>(n));
            k_scan_count<<<nscan, kThreads, 0, st>>>(n, e->flags.p, 3, e->scan_counts.p);
            k_scan_blocks<<<1, 1024, 0, st>>>(nscan, e->scan_counts.p, e->scan_total.p);
            k_scan_scatter<<<nscan, kThreads, 0, st>>>(n, e->flags.p, 3, e->scan_counts.p, e->act.p);
            CK(cudaMemcpyAsync(&m, e->scan_total.p, sizeof(int), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            CK(cudaGetLastError());
            if (m <= 0)
            {
                // the reference leaves an EMPTY grid here (clearVoxelsOutsideThinShell erases everything; the following lighting estimate
                // then fails and Intrinsic3D::refine skips the level): same state, not an error
                e->n = 0; e->have_sh = false; e->have_iter = false; e->shard_ready = false; e->sv_S = 0; e->sv_x = nullptr;
                collect_kernel_times(e);
                if (num_voxels_out) *num_voxels_out = 0;
                return 0;
            }
            // the spare set is grown to at least the capacity of the set it will be swapped with: capacities never shrink, so a later
            // i3d_upload_grid of the original size does not reallocate (measured: 279 ms of cudaFree/cudaMalloc on every second call
            // of a prune -> upload cycle, profiles/r02r_refine_level_stages.log)
            nx.ensure(std::max<size_t>(m, e->x.cap)); ny.ensure(std::max<size_t>(m, e->y.cap)); nz.ensure(std::max<size_t>(m, e->z.cap));
            nsdf0.ensure(std::max<size_t>(m, e->sdf0.cap)); nsdf.ensure(std::max<size_t>(m, e->sdfA.cap)); nalb.ensure(std::max<size_t>(m, e->albA.cap));
            nw.ensure(std::max<size_t>(m, e->weight.cap)); nrgb.ensure(std::max<size_t>(m, e->rgb.cap));
            VoxelArrays out{nx.p, ny.p, nz.p, nsdf0.p, nsdf.p, nalb.p, nw.p, nrgb.p};
            k_gather_voxels<<<blocks_for(static_cast<size_t>(m)), kThreads, 0, st>>>(m, e->act.p, g, out);
            CK(cudaStreamSynchronize(st));          // the old arrays become the spare set in the swap below
            if (install_grid(e, m, nx, ny, nz, nsdf0, nsdf, nalb, nw, nrgb)) return fail(e, "i3d_clear_voxels_outside_thin_shell: internal error (duplicate voxels)");
        }
        collect_kernel_times(e);
        if (num_voxels_out) *num_voxels_out = m;
        return 0;
    });
}

int i3d_upsample_grid(I3DEngine* e, int64_t* num_voxels_out)
{
    if (!e || e->n <= 0) return fail(e, "i3d_upsample_grid: upload the grid first");
    if (e->n > (1ll << 27)) return fail(e, "i3d_upsample_grid: %lld voxels would exceed the 2^30 voxel limit", static_cast<long long>(e->n));
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const int64_t n = e->n, m = 8 * n;
        e->timed.clear(); e->ev_used = 0; e->phases.erase("upsample");
        Dev<int32_t>&nx = e->sp_x, &ny = e->sp_y, &nz = e->sp_z; Dev<double>&nsdf0 = e->sp_sdf0, &nsdf = e->sp_sdf, &nalb = e->sp_alb; Dev<float>& nw = e->sp_w; Dev<uchar4>& nrgb = e->sp_rgb;
        {
            Timer t(e, "upsample", 0);
            const GridView g = e->grid_view(e->sdf, e->alb);
            nx.ensure(m); ny.ensure(m); nz.ensure(m); nsdf0.ensure(m); nsdf.ensure(m); nalb.ensure(m); nw.ensure(m); nrgb.ensure(m);
            VoxelArrays out{nx.p, ny.p, nz.p, nsdf0.p, nsdf.p, nalb.p, nw.p, nrgb.p};
            k_upsample<<<blocks_for(static_cast<size_t>(m)), kThreads, 0, st>>>(g, e->up_keys.p, e->up_vals.p, e->hash_cap - 1, out);
            CK(cudaStreamSynchronize(st));
            CK(cudaGetLastError());
            // SparseVoxelGrid::create(voxelSize * 0.5f): truncation = 5 * voxel size (src/sparse_voxel_grid.cpp:48)
            e->voxel_size = e->voxel_size * 0.5f; e->truncation = e->voxel_size * 5.0f;
            if (install_grid(e, m, nx, ny, nz, nsdf0, nsdf, nalb, nw, nrgb)) return fail(e, "i3d_upsample_grid: internal error (duplicate voxels)");
        }
        collect_kernel_times(e);
        if (num_voxels_out) *num_voxels_out = m;
        return 0;
    });
}

int i3d_download_grid(I3DEngine* e, int32_t* xyz, double* sdf0, double* sdf_refined, double* albedo, float* weight, uint8_t* rgb, float* voxel_size)
{
    if (!e || e->n <= 0) return fail(e, "i3d_download_grid: no grid");
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t n = static_cast<size_t>(e->n);
        if (xyz)
        {
            e->up_xyz.ensure(3 * n);
            k_interleave_xyz<<<blocks_for(n), kThreads, 0, st>>>(e->n, e->x.p, e->y.p, e->z.p, e->up_xyz.p);
            CK(cudaMemcpyAsync(xyz, e->up_xyz.p, 3 * n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        }
        if (sdf0) CK(cudaMemcpyAsync(sdf0, e->sdf0.p, n * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (sdf_refined) CK(cudaMemcpyAsync(sdf_refined, e->sdf, n * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (albedo) CK(cudaMemcpyAsync(albedo, e->alb, n * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (weight) CK(cudaMemcpyAsync(weight, e->weight.p, n * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (rgb)
        {
            e->up_rgb.ensure(3 * n);
            k_interleave_rgb<<<blocks_for(n), kThreads, 0, st>>>(e->n, e->rgb.p, e->up_rgb.p);
            CK(cudaMemcpyAsync(rgb, e->up_rgb.p, 3 * n, cudaMemcpyDeviceToHost, st));
        }
        CK(cudaStreamSynchronize(st));
        CK(cudaGetLastError());
        if (voxel_size) *voxel_size = e->voxel_size;
        return 0;
    });
}

int i3d_comm_unique_id(uint8_t id128[128])
{
    std::string err;
    if (!g_nccl.load(&err)) { g_create_error = err; return 1; }
    NcclApi::UniqueId id;
    if (g_nccl.GetUniqueId(&id) != 0) { g_create_error = "ncclGetUniqueId failed"; return 1; }
    std::memcpy(id128, id.internal, 128);
    return 0;
}

int i3d_comm_init(I3DEngine* e, int32_t rank, int32_t world, const uint8_t id128[128])
{
    if (!e) return 1;
    if (world <= 1) { e->rank = 0; e->world = 1; return 0; }
    std::string err;
    if (!g_nccl.load(&err)) return fail(e, "i3d_comm_init: %s", err.c_str());
    return guarded(e, [&]() {
        NcclApi::UniqueId id;
        std::memcpy(id.internal, id128, 128);
        NK(g_nccl.CommInitRank(&e->comm, world, id, rank));
        e->rank = rank; e->world = world; e->shard_ready = false;
        return 0;
    });
}

int i3d_comm_p2p_export(I3DEngine* e, uint8_t handle64[64])
{
    if (!e || !handle64) return 1;
    if (e->world <= 1) return fail(e, "i3d_comm_p2p_export: call i3d_comm_init (world > 1) first");
    return guarded(e, [&]() {
        static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
        const size_t bytes = 64ull << 20;
        e->p2p_ready = false;
        e->mbox.ensure(bytes);
        e->mbox_cap = (bytes - I3DEngine::kMboxFlagBytes) / (2 * sizeof(double));
        CK(cudaMemset(e->mbox.p, 0, I3DEngine::kMboxFlagBytes));
        cudaIpcMemHandle_t h;
        CK(cudaIpcGetMemHandle(&h, e->mbox.p));
        std::memcpy(handle64, &h, 64);
        return 0;
    });
}

int i3d_comm_p2p_connect(I3DEngine* e, const uint8_t* handles)
{
    if (!e || !handles) return 1;
    if (e->world <= 1 || !e->mbox.p) return fail(e, "i3d_comm_p2p_connect: call i3d_comm_p2p_export first");
    return guarded(e, [&]() {
        const int W = e->world;
        e->peer_base.assign(W, nullptr);
        std::vector<double*> hd(W);
        std::vector<unsigned int*> hf(W);
        for (int r = 0; r < W; ++r)
        {
            void* base = e->mbox.p;
            if (r != e->rank)
            {
                cudaIpcMemHandle_t h;
                std::memcpy(&h, handles + 64 * static_cast<size_t>(r), 64);
                CK(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
            }
            e->peer_base[r] = base;
            hf[r] = reinterpret_cast<unsigned int*>(base);
            hd[r] = reinterpret_cast<double*>(static_cast<uint8_t*>(base) + I3DEngine::kMboxFlagBytes);
        }
        e->d_peer_data.ensure(W); e->d_peer_flags.ensure(W);
        CK(cudaMemcpy(e->d_peer_data.p, hd.data(), W * sizeof(double*), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(e->d_peer_flags.p, hf.data(), W * sizeof(unsigned int*), cudaMemcpyHostToDevice));
        e->xseq = 0;
        e->p2p_ready = true;
        return 0;
    });
}

int i3d_set_shard(I3DEngine* e, int64_t voxel_begin, int64_t voxel_end)
{
    if (!e) return 1;
    if (e->n <= 0 || e->F <= 0) return fail(e, "i3d_set_shard: upload the grid and the frames first");
    if (voxel_begin < 0 || voxel_end > e->n || voxel_begin > voxel_end) return fail(e, "i3d_set_shard: bad range");
    e->shard_begin = voxel_begin; e->shard_end = voxel_end;
    if (e->world <= 1) return 0;
    return guarded(e, [&]() { return setup_shard(e); });
}

double i3d_phase_ms(const I3DEngine* e, const char* name)
{
    auto it = e->phases.find(name);
    return it == e->phases.end() ? 0.0 : it->second.ms;
}
int64_t i3d_phase_count(const I3DEngine* e, const char* name)
{
    auto it = e->phases.find(name);
    return it == e->phases.end() ? 0 : it->second.count;
}

int64_t i3d_debug_num_slots(const I3DEngine* e) { return e->have_iter ? static_cast<int64_t>(e->K) * e->stride : 0; }
int i3d_debug_set_kernel_timers(I3DEngine* e, int level)
{
    if (!e) return 1;
    e->timer_level = level > 0 ? 1 : 0;
    return 0;
}

int i3d_debug_set_keep_raw_jacobian(I3DEngine* e, int keep) { e->keep_raw = keep != 0; return 0; }

int i3d_debug_get_rows(I3DEngine* e, int32_t* voxel, int32_t* frame, double* residual, double* raw_weight, float* jac_colmajor)
{
    if (!e || !e->have_iter) return fail(e, "i3d_debug_get_rows: no iteration yet");
    return guarded(e, [&]() {
        const size_t S = static_cast<size_t>(e->K) * e->stride;
        cudaStream_t st = e->stream;
        if (voxel)
        {
            std::vector<int32_t> act(e->n_active);
            CK(cudaMemcpyAsync(act.data(), e->act.p, act.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            for (size_t i = 0; i < S; ++i) voxel[i] = -1;
            for (int k = 0; k < e->K; ++k) std::memcpy(voxel + static_cast<size_t>(k) * e->stride, act.data(), act.size() * sizeof(int32_t));
        }
        if (frame) CK(cudaMemcpyAsync(frame, e->row_frame.p, S * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (residual) CK(cudaMemcpyAsync(residual, e->row_res.p, S * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (raw_weight) CK(cudaMemcpyAsync(raw_weight, e->row_wraw.p, S * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (jac_colmajor) CK(cudaMemcpyAsync(jac_colmajor, e->J.p, I3D_EG_COLS * S * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        // the padding slots [n_active, stride) of every k are never written by the kernels: report them as "no row"
        for (int k = 0; k < e->K; ++k)
            for (int a = e->n_active; a < e->stride; ++a)
            {
                const size_t i = static_cast<size_t>(k) * e->stride + a;
                if (frame) frame[i] = -1;
                if (residual) residual[i] = 0.0;
                if (raw_weight) raw_weight[i] = 0.0;
            }
        return 0;
    });
}

int i3d_debug_get_observations(I3DEngine* e, int32_t K, int32_t* frames, float* weights, uint8_t* active)
{
    if (!e || !e->have_iter) return fail(e, "i3d_debug_get_observations: no iteration yet");
    if (K != e->K) return fail(e, "i3d_debug_get_observations: K mismatch");
    return guarded(e, [&]() {
        const size_t S = static_cast<size_t>(e->K) * e->stride;
        std::vector<int32_t> act(e->n_active), fr(S);
        std::vector<float> w(S);
        std::vector<uint8_t> fl(e->n);
        cudaStream_t st = e->stream;
        CK(cudaMemcpyAsync(act.data(), e->act.p, act.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (S) CK(cudaMemcpyAsync(fr.data(), e->obs_frame.p, S * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (S) CK(cudaMemcpyAsync(w.data(), e->obs_w.p, S * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(fl.data(), e->flags.p, e->n, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        for (int64_t v = 0; v < e->n; ++v)
        {
            if (active) active[v] = (fl[v] & FL_ACTIVE) ? 1 : 0;
            for (int k = 0; k < K; ++k) { if (frames) frames[v * K + k] = -1; if (weights) weights[v * K + k] = 0.0f; }
        }
        for (int a = 0; a < e->n_active; ++a)
        {
            // device slots are ordered by frame id; report in descending (weight, frame) priority
            std::vector<std::pair<std::pair<float, int>, int>> ord;
            for (int k = 0; k < K; ++k)
            {
                const size_t s = static_cast<size_t>(k) * e->stride + a;
                if (fr[s] >= 0) ord.push_back({{w[s], fr[s]}, k});
            }
            std::sort(ord.begin(), ord.end(), [](const auto& x, const auto& y) { return x.first > y.first; });
            for (size_t k = 0; k < ord.size(); ++k)
            {
                if (frames) frames[static_cast<size_t>(act[a]) * K + k] = ord[k].first.second;
                if (weights) weights[static_cast<size_t>(act[a]) * K + k] = ord[k].first.first;
            }
        }
        return 0;
    });
}

int i3d_debug_get_step(I3DEngine* e, double* step, uint8_t* free_mask, double* col_scale)
{
    if (!e || !e->have_iter) return fail(e, "i3d_debug_get_step: no iteration yet");
    return guarded(e, [&]() {
        const size_t U = static_cast<size_t>(e->U());
        std::vector<float> d(U), s(U);
        CK(cudaMemcpyAsync(d.data(), e->v_delta.p, U * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaMemcpyAsync(s.data(), e->v_s.p, U * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        for (size_t j = 0; j < U; ++j)
        {
            if (step) step[j] = d[j];
            if (free_mask) free_mask[j] = s[j] != 0.0f;
            if (col_scale) col_scale[j] = s[j];
        }
        return 0;
    });
}

int i3d_debug_get_normal_equations(I3DEngine* e, float* b, float* s, float* jtj, float* cam_acc)
{
    if (!e || !e->have_iter) return fail(e, "i3d_debug_get_normal_equations: no iteration yet");
    return guarded(e, [&]() {
        const size_t U = static_cast<size_t>(e->U());
        cudaStream_t st = e->stream;
        if (b) CK(cudaMemcpyAsync(b, e->v_b.p, U * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (s) CK(cudaMemcpyAsync(s, e->v_s.p, U * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (jtj) CK(cudaMemcpyAsync(jtj, e->v_jtj.p, U * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (cam_acc) CK(cudaMemcpyAsync(cam_acc, e->cam_acc.p, CamAccLayout{e->F}.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    });
}

int i3d_debug_apply_operator(I3DEngine* e, const float* v, float* q)
{
    if (!e || !e->have_iter) return fail(e, "i3d_debug_apply_operator: no iteration yet");
    if (!v || !q) return fail(e, "i3d_debug_apply_operator: NULL vector");
    if (e->world > 1) return fail(e, "i3d_debug_apply_operator: single GPU only");
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t U = static_cast<size_t>(e->U());
        const I3DParams& P = e->last_params;
        e->dbg_v.ensure(U);
        // the operator kernels are no-ops once the PCG has stopped: run them under a running copy of the control block and
        // put the original back afterwards (with is_cg_iteration = 0 they do not write it)
        CgCtl saved{}, running{};
        CK(cudaMemcpyAsync(&saved, e->ctl.p, sizeof(CgCtl), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        running = saved; running.done = 0; running.inv_radius = 0.0;
        CK(cudaMemcpyAsync(e->ctl.p, &running, sizeof(CgCtl), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(e->dbg_v.p, v, U * sizeof(float), cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(e->v_qg.p, 0, U * sizeof(float), st));
        const int timer_level = e->timer_level;
        const int64_t launches = e->launches;
        e->timer_level = -1;                       // keep the last iteration's kernel table
        GridView g = e->grid_view(e->sdf, e->alb);
        RegView rv;
        rv.flags = e->flags.p; rv.ea_w = e->ea_w.p; rv.lap = e->lap.p;
        rv.use_er = P.use_er; rv.use_es = P.use_es; rv.use_ea = P.use_ea;
        EgRows rows;
        rows.n_active = e->n_active; rows.K = e->K; rows.stride = e->stride; rows.act = e->act.p; rows.J = e->J.p; rows.row_frame = e->row_frame.p;
        rows.row_res = e->row_res.p; rows.row_wraw = e->row_wraw.p; rows.row_w = e->row_w.p;
        const SolveVecs sv = solve_vecs(e);
        const Shard sh = e->shard();
        const int64_t hc = e->held_count();
        pdl_launch(e, k_scale_vec, blocks_for(static_cast<size_t>(hc)), kThreads, 0, sv, sh, hc, e->dbg_v.p, 1.0f, sv.ps, e->ctl.p, 0);
        launch_operator(e, g, rv, rows, sv, sh, e->dbg_v.p, 0.0f, 0.0f, 0);
        e->timer_level = timer_level;
        e->launches = launches;
        std::vector<float> qg(U), s(U);
        CK(cudaMemcpyAsync(qg.data(), e->v_qg.p, U * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(s.data(), e->v_s.p, U * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaMemsetAsync(e->v_qg.p, 0, U * sizeof(float), st));      // k_op_partial cleared qgd
        CK(cudaMemcpyAsync(e->ctl.p, &saved, sizeof(CgCtl), cudaMemcpyHostToDevice, st));
        CK(cudaStreamSynchronize(st));
        CK(cudaGetLastError());
        for (size_t j = 0; j < U; ++j) q[j] = s[j] * qg[j];       // k_cg_update's q_j = s_j qg_j, without D^2
        return 0;
    });
}

} // extern "C"
