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
#include <string>
#include <vector>

#include "../../include/i3d_c_api.h"
#include "i3d_kernels.cuh"
#include "i3d_lighting.cuh"
#include "i3d_recolor.cuh"
#include "i3d_gridops.cuh"
#include "i3d_host.h"
#include "i3d_frames.h"
#include "i3d_fusion.h"
#include "i3d_mesh.h"
#include "i3d_render.h"
#include "i3d_texture.h"
#include "i3d_distance.h"
#include "i3d_grid_from_mesh.h"
#include "i3d_raster.h"
#include "i3d_track.h"

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

struct NcclError { int code; int line; };

enum Site { SITE_BUILD = 0, SITE_REG, SITE_FINISH, SITE_EG_APPLY, SITE_OP_POST, SITE_UPDATE, SITE_CAND, SITE_EG_COST, SITE_REG_COST, SITE_COUNT };
constexpr int kSiteVals = 9;
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
    Dev<float> obs_w;
    Dev<float4> Jt;                  // E_g rows, layout in EgRows
    Dev<float2> Jtail;
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
    Timing timing;               // the phase and kernel timers of every entry point
    int64_t launches = 0;        // kernels launched during the last i3d_gn_iteration (counted by pdl_launch; other entry points do not count)
    int64_t host_syncs = 0;      // cudaStreamSynchronize calls of the last i3d_gn_iteration
    Dev<IterDev> iter_dev;       // device-resident result / LM state of the current iteration
    int last_cg_iterations = 4, prev_cg_iterations = 4;  // PCG iteration counts of the previous two solves: their maximum sizes the first launch batch
    bool pcg_fused = true;       // k_cg_step where it applies (I3D_PCG_FUSED=0 at engine creation: the four-kernel chain)
    int64_t step_n = -1;         // grid size k_cg_step's launch shape was planned for (step_grid = 0: does not fit)
    unsigned step_grid = 0; int step_K = 0; size_t step_smem = 0;
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
    SubvolGrid sv_grid{};              // the subvolume table of the last estimate (sv_table), valid while sv_S > 0
    FusionState fusion;                // RGB-D fusion in progress (i3d_fusion.cu)
    ScoreScratch scores;               // keyframe scores (i3d_frames.cu)
    RgbdStore rgbd;                    // RGB-D frame store (i3d_frames.cu)
    SensorStore sensor;                // sensor store (i3d_frames.cu)
    MeshState mesh;                    // surface extraction (i3d_mesh.cu)
    TextureState tex;                  // texture of the resident mesh (i3d_texture.cu)
    DistanceState dist;                // reference mesh and distance results (i3d_distance.cu)
    GridFromMeshState gfm;             // the voxel grid from a mesh (i3d_grid_from_mesh.cu)
    RenderState render;                // keyframe renderer (i3d_render.cu)
    RasterState raster;                // rasterizer of the resident mesh (i3d_raster.cu)
    I3DShLighting relight{I3D_SH_ESTIMATE, 0, {}};     // lighting of the relit colour source (i3d_set_relight)
    TrackScratch track;                // frame-to-model tracker (i3d_render.cu)
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
        const char* file = std::strrchr(ce.file, '/') ? std::strrchr(ce.file, '/') + 1 : ce.file;     // the file name, without its directory
        return fail(e, "CUDA error %d (%s) at %s:%d: %s", static_cast<int>(ce.code), cudaGetErrorString(ce.code), file, ce.line, ce.what);
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

// Forgets everything derived from the voxel set: the per-voxel SH and the lighting estimate, the last iteration, the shard state and
// range, the resident mesh with its texture and raster planes, and the renderer's voxel box, brick bitmap and planes.  Every change of
// the voxel set calls it.
void forget_voxel_set(I3DEngine* e)
{
    e->have_sh = false; e->sv_S = 0; e->sv_x = nullptr; e->have_iter = false; e->mesh.have_mesh = false; e->tex.have = false;
    e->raster.have = false;
    e->render.box_ready = false; e->render.have_bricks = false; e->render.have_render = false;
    e->shard_ready = false; e->shard_begin = 0; e->shard_end = -1;
}

// Replaces the voxel set by the m voxels that `fill` writes into the spare arrays (VoxelArrays, on e->stream), then swaps the two sets
// and rebuilds the topology.  The spare set is grown to at least the capacity of the set it will be swapped with: capacities never
// shrink, so a later i3d_upload_grid of the original size does not reallocate (measured: 279 ms of cudaFree/cudaMalloc on every second
// call of a prune -> upload cycle, profiles/r02r_refine_level_stages.log).  Returns non-zero if two voxels share coordinates.
template <class Fill>
int install_grid(I3DEngine* e, int64_t m, Fill&& fill)
{
    const size_t cnt = static_cast<size_t>(m);
    auto grow = [cnt](auto& spare, const auto& live) { spare.ensure(std::max(cnt, live.cap)); };
    grow(e->sp_x, e->x); grow(e->sp_y, e->y); grow(e->sp_z, e->z);
    grow(e->sp_sdf0, e->sdf0); grow(e->sp_sdf, e->sdfA); grow(e->sp_alb, e->albA); grow(e->sp_w, e->weight); grow(e->sp_rgb, e->rgb);
    fill(VoxelArrays{e->sp_x.p, e->sp_y.p, e->sp_z.p, e->sp_sdf0.p, e->sp_sdf.p, e->sp_alb.p, e->sp_w.p, e->sp_rgb.p});
    CK(cudaStreamSynchronize(e->stream));          // the old arrays become the spare set in the swap below
    CK(cudaGetLastError());
    e->x.swap(e->sp_x); e->y.swap(e->sp_y); e->z.swap(e->sp_z); e->sdf0.swap(e->sp_sdf0); e->sdfA.swap(e->sp_sdf); e->albA.swap(e->sp_alb);
    e->weight.swap(e->sp_w); e->rgb.swap(e->sp_rgb);
    e->n = m;
    e->sdfB.ensure(cnt); e->albB.ensure(cnt);
    e->sdf = e->sdfA.p; e->c_sdf = e->sdfB.p; e->alb = e->albA.p; e->c_alb = e->albB.p;
    forget_voxel_set(e);
    return rebuild_topology(e);
}

// Installs F frames of W x H as the engine's luminance / depth planes at scale pyr_scale: `fill` writes e->lum / e->depth (sized here) on
// e->stream.  The one place that knows what a frame change invalidates: a new frame count drops the camera and the last iteration, a new
// size drops the colour planes, the depth tiles of the frame culling are rebuilt, and the planes of the last render and of the last
// keyframe rasterization are dropped.
template <class Fill>
void install_frames(I3DEngine* e, int32_t F, int32_t W, int32_t H, double pyr_scale, Fill&& fill)
{
    const size_t cnt = static_cast<size_t>(F) * W * H;
    e->render.have_render = false;
    if (e->raster.keyframes) e->raster.have = false;
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
    fill();
    {
        const int TW = (W + kCullTile - 1) / kCullTile, TH = (H + kCullTile - 1) / kCullTile;
        const size_t nt = static_cast<size_t>(F) * TW * TH;
        e->tile_min.ensure(nt); e->tile_max.ensure(nt);
        k_depth_tiles<<<static_cast<unsigned>(nt), 256, 0, e->stream>>>(F, W, H, e->depth.p, e->tile_min.p, e->tile_max.p);
    }
}

// A camera the fusion and resizeDepth can use: a positive size and finite intrinsics with fx, fy > 0
bool pinhole_ok(const I3DFusionCamera* c)
{
    return c && c->width > 0 && c->height > 0 && c->fx > 0.0f && c->fy > 0.0f && std::isfinite(c->fx) && std::isfinite(c->fy) &&
           std::isfinite(c->cx) && std::isfinite(c->cy);
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

EgRows eg_rows(I3DEngine* e)
{
    EgRows rows;
    rows.n_active = e->n_active; rows.K = e->K; rows.stride = e->stride; rows.act = e->act.p; rows.Jt = e->Jt.p; rows.Jtail = e->Jtail.p;
    rows.row_frame = e->row_frame.p; rows.row_res = e->row_res.p; rows.row_wraw = e->row_wraw.p;
    return rows;
}

RegView reg_view(I3DEngine* e, const I3DParams& P)
{
    RegView rv;
    rv.flags = e->flags.p; rv.ea_w = e->ea_w.p; rv.lap = e->lap.p;
    rv.use_er = P.use_er; rv.use_es = P.use_es; rv.use_ea = P.use_ea;
    return rv;
}

// The camera of the frame scans (k_select_obs, k_recolor) from the intrinsics and distortion hc9 read back from e->cam: intrinsics *
// pyr_scale cast to float (optimizer.cpp:124-127; Camera::setIntrinsics).  The caller reads hc9 back, so that the GN iteration can
// read it in the same synchronisation as its row count.
SelectCam select_cam(const I3DEngine* e, const double hc9[9], float occlusion)
{
    SelectCam sc;
    sc.fx = static_cast<float>(hc9[0] * e->pyr_scale); sc.fy = static_cast<float>(hc9[1] * e->pyr_scale);
    sc.cx = static_cast<float>(hc9[2] * e->pyr_scale); sc.cy = static_cast<float>(hc9[3] * e->pyr_scale);
    sc.dist_zero = 1;
    for (int k = 0; k < 5; ++k) { sc.d[k] = static_cast<float>(hc9[4 + k]); if (sc.d[k] != 0.0f) sc.dist_zero = 0; }
    sc.occlusion = occlusion;
    return sc;
}

// The conservative frame culling of the frame scans.  I3D_NO_CULL visits every frame: the results must not change.
CullView cull_view(const I3DEngine* e, unsigned long long* stats)
{
    static const bool no_cull = std::getenv("I3D_NO_CULL") != nullptr;
    return CullView{e->tile_min.p, e->tile_max.p, no_cull ? 0 : 1, stats};
}

#define NK(call)                                                            \
    do {                                                                    \
        int _r = (call);                                                    \
        if (_r != 0) throw NcclError{_r, __LINE__};                         \
    } while (0)


// I3D_PDL=0 launches without programmatic dependent launch, to rule out ordering races
bool pdl_enabled() { static const bool on = [] { const char* v = std::getenv("I3D_PDL"); return !(v && v[0] == '0'); }(); return on; }

// Every kernel of the Gauss-Newton iteration is launched here, and counted in e->launches.  It is launched with programmatic stream
// serialization (programmatic dependent launch): the kernels begin with griddepcontrol.wait (pdl_prologue(), i3d_kernels.cuh), so the
// next grid's launch latency overlaps the tail of its predecessor instead of following it.  I3D_PDL=0 disables the attribute (the
// device-side wait is then a no-op).  COOPERATIVE: a cooperative launch (grid barriers, k_cg_step); the two attributes combine.
template <bool COOPERATIVE = false, class... KArgs, class... Args>
void pdl_launch(I3DEngine* e, void (*kern)(KArgs...), unsigned grid, unsigned block, size_t smem, Args&&... args)
{
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = e->stream;
    cudaLaunchAttribute at[2];
    unsigned na = 0;
    if (COOPERATIVE) { at[na].id = cudaLaunchAttributeCooperative; at[na].val.cooperative = 1; ++na; }
    if (pdl_enabled()) { at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
    cfg.attrs = at; cfg.numAttrs = na;
    CK(cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...));
    e->launches += 1;
}

// k_eg_rows variant selection.  Cost evaluation (ROWS_COST): the pose table of all F frames is staged into shared memory by a bulk-async
// copy (256 threads, 2 blocks per SM) when two blocks with their per-voxel state and the table fit into the SM's shared memory —
// measured at C3: 0.455 ms staged vs 0.486 ms from L1.  Jacobian build (ROWS_BUILD): 128 threads x 4 blocks, poses from L1 — the
// staged variant was SLOWER there (0.800 vs 0.719 ms: the 40-float derivative state per thread makes the 256-thread blocks 108 KB
// each, and the block-granular tail costs more than the L1 misses it removes).  profiles/r02p_*.json.
template <int MODE>
void launch_eg_rows(I3DEngine* e, const GridView& g, const CamView& cv, const EgRows& rows, const int32_t* obs_frame, const float* obs_w)
{
    if constexpr (MODE == ROWS_COST)
    {
        const size_t smem = rows_smem_bytes(MODE, 256, true, e->F);
        if (2 * (smem + 1024) <= 227u * 1024u)
        {
            auto kern = k_eg_rows<MODE, 256, true>;
            CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
            pdl_launch(e, kern, blocks_for(static_cast<size_t>(rows.stride), 256), 256, smem, g, e->frame_view(), cv, rows, obs_frame, obs_w, e->site(SITE_EG_COST));
            return;
        }
    }
    auto kern = k_eg_rows<MODE, 128, false>;
    const size_t smem = rows_smem_bytes(MODE, 128, false, e->F);
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    pdl_launch(e, kern, blocks_for(static_cast<size_t>(rows.stride), 128), 128, smem, g, e->frame_view(), cv, rows, obs_frame, obs_w, e->site(SITE_EG_COST));
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
        return;
    }
    NK(g_nccl.AllReduce(dev, dev, static_cast<size_t>(count), NCCL_FLOAT64, NCCL_SUM, e->comm, e->stream));
    if (kind >= 0) pdl_launch(e, k_epilogue, 1, 32, 0, e->ctl.p, dev, kind, respect_done);
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
        return;
    }
    e->xbuf.ensure(2 * static_cast<size_t>(e->n_shared) + CamAccLayout{e->F}.size() + 64);
    pdl_launch(e, k_pack, blocks_for(threads), kThreads, 0, shv, v0, v1, extra_f, n_extra_f, extra_d, n_extra_d, e->xbuf.p, e->ctl.p, respect_done);
    NK(g_nccl.AllReduce(e->xbuf.p, e->xbuf.p, total, NCCL_FLOAT64, NCCL_SUM, e->comm, e->stream));
    pdl_launch(e, k_unpack, blocks_for(threads), kThreads, 0, shv, v0, v1, extra_f, n_extra_f, extra_d, n_extra_d, e->xbuf.p, e->ctl.p, respect_done);
    if (epilogue_kind >= 0) pdl_launch(e, k_epilogue, 1, 32, 0, e->ctl.p, extra_d, epilogue_kind, respect_done);
}

size_t apply_smem_bytes(int F, int K)
{
    return static_cast<size_t>((6 * F + 9 + 15) & ~15) * sizeof(double) + static_cast<size_t>(14 + 6 * K) * kThreads * sizeof(float);
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
    CK(cudaFuncGetAttributes(&fa_app, k_eg_apply));
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
void launch_eg_apply(I3DEngine* e, const GridView& g, const RegView& rv, const EgRows& rows, const SolveVecs& sv)
{
    if (rows.n_active == 0) return;
    Timer kt(e->timing, e->stream, "k_eg_apply");     // the dominant kernel: every launch is timed (roofline = true average)
    pdl_launch(e, k_eg_apply, blocks_for(rows.n_active), kThreads, apply_smem_bytes(e->F, rows.K), g, rows, rv, sv, sv.ps, e->ctl.p, e->site(SITE_EG_APPLY));
}

void launch_operator(I3DEngine* e, const GridView& g, const RegView& rv, const EgRows& rows, const SolveVecs& sv, const Shard& sh, const float* vin,
                     float dmin, float dmax, int is_cg_iteration)
{
    launch_eg_apply(e, g, rv, rows, sv);
    {
        Timer kt(e->timing, e->stream, "k_op_partial", 1);
        pdl_launch(e, k_op_partial, blocks_for(static_cast<size_t>((e->held_count() + 3) / 4)), kThreads, 0,
            g, rv, sv, sh, e->held_count(), vin, sv.ps, e->type_w.p, dmin, dmax, e->ctl.p, e->site(SITE_OP_POST), e->site(SITE_EG_APPLY).out, is_cg_iteration);
    }
    if (e->world > 1)
    {
        Timer kt(e->timing, e->stream, "exchange", 1);
        exchange(e, sv.qg, nullptr, sv.qg + 2 * e->n, 6 * e->F + 9, e->site(SITE_OP_POST).out, 1, 1, is_cg_iteration ? EPI_OPERATOR_CG : -1);
    }
}

// Launch shape of k_cg_step for the current grid: the most blocks per SM at which every block is resident together with its
// K = ceil(items / threads) shared-memory slots.  Returns false (the four-kernel chain runs) when no shape fits.
bool plan_cg_step(I3DEngine* e)
{
    if (e->step_n == e->n) return e->step_grid > 0;
    e->step_n = e->n; e->step_grid = 0;
    int sms = 0, optin = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, e->device));
    CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, e->device));
    cudaFuncAttributes fa0{}, fa1{};
    CK(cudaFuncGetAttributes(&fa0, k_cg_step<false>));
    CK(cudaFuncGetAttributes(&fa1, k_cg_step<true>));
    const size_t dyn_max = static_cast<size_t>(optin) - std::max(fa0.sharedSizeBytes, fa1.sharedSizeBytes);
    CK(cudaFuncSetAttribute(k_cg_step<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(dyn_max)));
    CK(cudaFuncSetAttribute(k_cg_step<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(dyn_max)));
    const int64_t items = (e->n + 3) / 4;
    for (int bps = 2048 / kStepThreads; bps >= 1; --bps)
    {
        const int64_t threads = static_cast<int64_t>(bps) * sms * kStepThreads;
        const int64_t K = (items + threads - 1) / threads;
        const size_t smem = static_cast<size_t>(K) * kStepSlots * kStepThreads * sizeof(float);
        if (smem > dyn_max) break;
        int occ0 = 0, occ1 = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ0, k_cg_step<false>, kStepThreads, smem));
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ1, k_cg_step<true>, kStepThreads, smem));
        if (std::min(occ0, occ1) < bps) continue;
        if (static_cast<size_t>(bps) * sms + 8 > e->max_blocks) break;     // block partials live in the reduction scratch
        e->step_grid = static_cast<unsigned>(bps * sms); e->step_K = static_cast<int>(K); e->step_smem = smem;
        return true;
    }
    return false;
}

// k_cg_step is a cooperative launch (grid barriers between its phases); it keeps programmatic stream serialization like every other
// kernel of the iteration: its blocks wait in griddepcontrol.wait until k_eg_apply has finished.
template <bool INIT>
void launch_cg_step(I3DEngine* e, const GridView& g, const RegView& rv, const SolveVecs& sv, float dmin, float dmax)
{
    const int64_t items = (e->n + 3) / 4;
    pdl_launch<true>(e, k_cg_step<INIT>, e->step_grid, kStepThreads, e->step_smem, g, rv, sv, items, e->step_K, e->type_w.p, e->minv.p, dmin, dmax,
                     e->ctl.p, e->site(SITE_OP_POST), e->site(SITE_EG_APPLY).out, e->site(SITE_UPDATE));
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
    e->timing.phases.clear(); begin_timing(e->timing, {}); e->launches = 0; e->host_syncs = 0;        // the iteration owns every phase
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
    Timer t_total(e->timing, e->stream, "total");
    auto sync = [&]() { CK(cudaStreamSynchronize(st)); e->host_syncs += 1; };

    // ------------------------------------------------------------------ activity, compaction of the rows this rank owns
    Timer t_sel(e->timing, e->stream, "select");
    e->flags.ensure(n);
    GridView g = e->grid_view(e->sdf, e->alb);
    // flags over the range this rank reads (own voxels + 4 stencil rings); compaction of the owned rows over the owned range
    pdl_launch(e, k_flags, blocks_for(static_cast<size_t>(sh.loc_end - sh.loc_begin)), kThreads, 0, g, sh, P.thres_shell, P.fix_all_albedo, e->flags.p);
    const int nscan = std::max(1, static_cast<int>((own + kScanChunk - 1) / kScanChunk));
    e->scan_counts.ensure(nscan); e->scan_total.ensure(1); e->act.ensure(n);
    pdl_launch(e, k_scan_count, nscan, kThreads, 0, own, e->flags.p + sh.own_begin, FL_ROW, e->scan_counts.p);
    pdl_launch(e, k_scan_blocks, 1, 1024, 0, nscan, e->scan_counts.p, e->scan_total.p);
    pdl_launch(e, k_scan_scatter, nscan, kThreads, 0, own, e->flags.p + sh.own_begin, FL_ROW, e->scan_counts.p, e->act.p, static_cast<int32_t>(sh.own_begin));
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
    int32_t n_active = 0;
    double hc9[9];
    CK(cudaMemcpyAsync(&n_active, e->scan_total.p, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(hc9, e->cam + 6 * static_cast<size_t>(F), 9 * sizeof(double), cudaMemcpyDeviceToHost, st));      // select_cam()
    sync();
    e->n_active = n_active;
    const int stride = (n_active + 63) & ~63;          // slots per k: keeps every J column segment 256 B aligned
    e->stride = stride;
    const size_t S = static_cast<size_t>(K) * stride;

    // ------------------------------------------------------------------ k1 observation selection
    e->obs_frame.ensure(S + 1); e->obs_w.ensure(S + 1);
    if (n_active > 0)
    {
        const SelectCam sc = select_cam(e, hc9, P.occlusion_distance);
        const size_t smem = 12 * static_cast<size_t>(F) * sizeof(float);
        auto kern = (K <= 5) ? k_select_obs<5> : k_select_obs<I3D_MAX_OBS>;
        if (smem > 48 * 1024) CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        Timer kt(e->timing, e->stream, "k_select_obs");
        static const bool want_stats = std::getenv("I3D_CULL_STATS") != nullptr;
        e->cull_stats.ensure(2);
        if (want_stats) CK(cudaMemsetAsync(e->cull_stats.p, 0, 2 * sizeof(unsigned long long), st));
        const CullView cull = cull_view(e, want_stats ? e->cull_stats.p : nullptr);
        pdl_launch(e, kern, blocks_for(static_cast<size_t>(n_active)), kThreads, smem, g, e->frame_view(), e->Rt.p, sc, cull, n_active, stride, e->act.p, K,
                                                                                e->obs_frame.p, e->obs_w.p);
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
    Timer t_build(e->timing, e->stream, "build");
    e->Jt.ensure(EgRows::kTiles * S + 1); e->Jtail.ensure(S + 1);
    e->row_frame.ensure(S + 1); e->row_res.ensure(S + 1); e->row_wraw.ensure(S + 1);
    e->ea_w.ensure(3 * static_cast<size_t>(n)); e->lap.ensure(n);
    // set unconditionally: the default limit is 48 KB minus the kernel's static shared memory, not 48 KB
    CK(cudaFuncSetAttribute(k_eg_apply, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(apply_smem_bytes(F, K))));
    const EgRows rows = eg_rows(e);
    CamView cv{e->cam, e->pose_ctx.p, F};
    if (n_active > 0)
    {
        {
            Timer kt(e->timing, e->stream, "k_eg_build");
            launch_eg_rows<ROWS_BUILD>(e, g, cv, rows, e->obs_frame.p, e->obs_w.p);
        }
        const size_t smem = accum_smem_bytes(F, K);
        if (smem > 48 * 1024) CK(cudaFuncSetAttribute(k_eg_accum, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        {
            Timer kt(e->timing, e->stream, "k_eg_accum", 1);
            pdl_launch(e, k_eg_accum, blocks_for(static_cast<size_t>(n_active)), kThreads, smem, g, rows, F, e->v_bgd.p, e->v_cgd.p, e->cam_accd.p, e->site(SITE_BUILD));
        }
        pdl_launch(e, k_acc_to_float, blocks_for(std::max(U, static_cast<size_t>(lay.size()))), kThreads, 0, static_cast<int64_t>(U), lay.size(),
                   e->v_bgd.p, e->v_cgd.p, e->cam_accd.p, e->v_bg.p, e->v_cg.p, e->cam_acc.p);
    }
    const RegView rv = reg_view(e, P);
    pdl_launch(e, k_reg_build, blocks_for(static_cast<size_t>((sh.loc_end - sh.loc_begin + 3) / 4)), kThreads, 0, g, rv, sh, e->site(SITE_REG));
    {
        // active-voxel count rides along in the unused tail of SITE_BUILD
        const double na = static_cast<double>(n_active);
        CK(cudaMemcpyAsync(e->site(SITE_BUILD).out + 3, &na, sizeof(double), cudaMemcpyHostToDevice, st));
    }
    if (multi) exchange(e, e->v_bg.p, e->v_cg.p, e->cam_acc.p, lay.size(), e->red_out.p, 2 * kSiteVals, 0);   // SITE_BUILD + SITE_REG are adjacent
    // NLSSolver::normalizeCostTermWeights (nls_solver.cpp:379-394) on the device
    pdl_launch(e, k_type_weights, 1, 32, 0, e->iter_dev.p, e->site(SITE_BUILD).out, e->site(SITE_REG).out, P, n, e->type_w.p);
    if (S > 0) pdl_launch(e, k_row_weights, blocks_for(S), kThreads, 0, rows, e->type_w.p);
    SolveVecs sv = solve_vecs(e);
    pdl_launch(e, k_finish_problem, blocks_for(static_cast<size_t>((hc + 3) / 4)), kThreads, 0, g, rv, sv, sh, hc, e->type_w.p, e->cam_acc.p, P.fix_poses, P.fix_intrinsics,
                                                                              P.fix_distortion, P.gradient_tolerance, e->site(SITE_FINISH), e->cam);
    allreduce_scalars(e, e->site(SITE_FINISH).out, 3, -1, 0);
    pdl_launch(e, k_iter_finish, 1, 32, 0, e->iter_dev.p, e->site(SITE_FINISH).out, P);
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
    Timer t_solve(e->timing, e->stream, "solve");
    const float dmin = static_cast<float>(P.min_lm_diagonal), dmax = static_cast<float>(std::min(P.max_lm_diagonal, 3.0e38));
    // voxel unknowns of the held hull: 4 per thread (16 B accesses); the first F + 2 threads take one camera block each
    const unsigned upd_blocks = blocks_for(static_cast<size_t>((sh.held_voxel_unknowns() + 3) / 4 + F + 2));
    auto launch_update = [&](bool init, int refresh) {
        if (init) pdl_launch(e, k_cg_update<true>, upd_blocks, kThreads, 0, sv, sh, e->minv.p, dmin, dmax, e->ctl.p, refresh, e->site(SITE_UPDATE));
        else pdl_launch(e, k_cg_update<false>, upd_blocks, kThreads, 0, sv, sh, e->minv.p, dmin, dmax, e->ctl.p, refresh, e->site(SITE_UPDATE));
    };
    const unsigned vec_blocks = blocks_for(static_cast<size_t>(hc));
    const int max_it = P.forced_cg_iterations > 0 ? P.forced_cg_iterations : P.max_linear_solver_iterations;
    // single GPU: the per-unknown half of a PCG iteration is one cooperative k_cg_step (operator finish, update, next direction)
    const bool fused = e->pcg_fused && !multi && plan_cg_step(e);
    int enq = 0;                 // PCG iterations enqueued in the current trial
    bool dir_ready = false;      // p and ps of the next iteration were formed by the k_cg_step before it
    auto enqueue_pcg = [&](int count) {
        for (int bidx = 0; bidx < count && enq < max_it; ++bidx)
        {
            ++enq;
            const bool refresh = (enq % P.residual_reset_period == 0);
            if (!dir_ready)
            {
                Timer kt(e->timing, e->stream, "k_cg_dir", 1);
                pdl_launch(e, k_cg_dir4, blocks_for(static_cast<size_t>((hc + 3) / 4)), kThreads, 0, sv, sh, hc, e->ctl.p);
            }
            dir_ready = false;
            if (fused && !refresh)
            {
                launch_eg_apply(e, g, rv, rows, sv);
                Timer kt(e->timing, e->stream, "k_cg_update", 1);        // k_cg_step is timed in k_cg_update's place
                launch_cg_step<false>(e, g, rv, sv, dmin, dmax);
                dir_ready = true;
                continue;
            }
            launch_operator(e, g, rv, rows, sv, sh, sv.p, dmin, dmax, 1);
            if (refresh)
            {
                // exact residual: x += alpha p ; r = b - A x   (needs the operator's qg consumed first: do the plain update
                // of x only, then apply the operator to x)
                pdl_launch(e, k_x_update, vec_blocks, kThreads, 0, sv, sh, hc, e->ctl.p);
                // discard A p: k_cg_update(refresh) below consumes A x, so clear qg by a dry consume
                CK(cudaMemsetAsync(e->v_qg.p, 0, U * sizeof(float), st));
                pdl_launch(e, k_scale_vec, vec_blocks, kThreads, 0, sv, sh, hc, sv.x, 1.0f, sv.ps, e->ctl.p, 1);
                launch_operator(e, g, rv, rows, sv, sh, sv.x, dmin, dmax, 0);
                launch_update(false, 1);
            }
            else
            {
                Timer kt(e->timing, e->stream, "k_cg_update", 1);
                launch_update(false, 0);
            }
            if (multi) allreduce_scalars(e, e->site(SITE_UPDATE).out, 3, EPI_UPDATE, 1);
        }
    };
    // candidate point + candidate cost + the trust-region decision, all stream-ordered behind the PCG.  The model cost change comes
    // from the PCG's own scalars (k_lm_decide): no extra pass over the Jacobian.
    auto enqueue_decision = [&]() {
        Timer t_cand(e->timing, e->stream, "candidate");
        CK(cudaMemsetAsync(e->red_out.p + SITE_CAND * kSiteVals, 0, 3 * kSiteVals * sizeof(double), st));
        pdl_launch(e, k_candidate, vec_blocks, kThreads, 0, g, sv, sh, hc, 0, e->cam, e->c_sdf, e->c_alb, e->c_cam, e->v_delta.p, e->ctl.p, e->site(SITE_CAND));
        GridView gc = e->grid_view(e->c_sdf, e->c_alb);
        pdl_launch(e, k_frame_pose, blocks_for(F, 64), 64, 0, F, e->c_cam, e->pose_ctx_c.p);
        CamView cvc{e->c_cam, e->pose_ctx_c.p, F};
        if (n_active > 0)
        {
            Timer kt(e->timing, e->stream, "k_eg_cost");
            launch_eg_rows<ROWS_COST>(e, gc, cvc, rows, nullptr, nullptr);
        }
        pdl_launch(e, k_reg_cost, blocks_for(static_cast<size_t>(own)), kThreads, 0, gc, rv, sh, e->c_sdf, e->c_alb, e->site(SITE_REG_COST));
        if (multi) allreduce_scalars(e, e->red_out.p + SITE_CAND * kSiteVals, 3 * kSiteVals, -1, 0);   // SITE_CAND, SITE_EG_COST, SITE_REG_COST are adjacent
        pdl_launch(e, k_lm_decide, 1, 32, 0, e->iter_dev.p, e->ctl.p, e->fail_flag.p, e->site(SITE_CAND).out, e->site(SITE_EG_COST).out,
                                      e->site(SITE_REG_COST).out, e->type_w.p, P);
    };
    IterDev h{};
    for (int it = 1; it <= P.lm_steps; ++it)
    {
        Timer t_pcg(e->timing, e->stream, "pcg");
        pdl_launch(e, k_lm_begin, 1, 32, 0, e->iter_dev.p, e->ctl.p, e->fail_flag.p, P);
        pdl_launch(e, k_cam_precond, blocks_for(static_cast<size_t>(F) + 2, 64), 64, 0, sv, e->cam_acc.p, e->type_w.p, e->ctl.p, dmin, dmax, e->minv.p, e->fail_flag.p);
        if (fused) launch_cg_step<true>(e, g, rv, sv, dmin, dmax);
        else launch_update(true, 0);
        dir_ready = fused;
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
            Timer t_more(e->timing, e->stream, "pcg");
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

// ---- surface extraction, rendering and tracking (i3d_mesh.cu, i3d_render.cu) ----------------------
// The sdf a mesh is cut from, or a colour mode reads: 0 = sdf0, 1 = the refined sdf
int check_sdf_source(I3DEngine* e, const char* who, int32_t sdf_source)
{
    if (sdf_source != 0 && sdf_source != 1) return fail(e, "%s: sdf_source must be 0 (sdf0) or 1 (sdf_refined), got %d", who, sdf_source);
    return 0;
}

// The checks shared by the calls that take a colour mode (the grid and the sdf source are checked by the caller): a shading mode
// needs the subvolume SH of a lighting estimate of the current voxel set.
int check_color_mode(I3DEngine* e, const char* who, int32_t mode)
{
    if (mode < I3D_MESH_COLOR_VOXEL || mode >= I3D_MESH_COLOR_COUNT)
        return fail(e, "%s: color_mode must be in [0, %d], got %d", who, I3D_MESH_COLOR_COUNT - 1, mode);
    if ((mode == I3D_MESH_COLOR_SHADING_SV || mode == I3D_MESH_COLOR_SHADING_SV_CONST) && (e->sv_S <= 0 || !e->sv_x))
        return fail(e, "%s: the shading modes need a lighting estimate of the current grid (i3d_estimate_lighting)", who);
    return 0;
}

// A lighting the decomposition and the relit raster can use: a known source, finite global coefficients, and for the estimate a lighting
// estimate of the current voxel set (the shading modes' rule)
int check_sh_lighting(I3DEngine* e, const char* who, const I3DShLighting& l)
{
    if (l.source != I3D_SH_ESTIMATE && l.source != I3D_SH_GLOBAL)
        return fail(e, "%s: the lighting source must be %d (estimate) or %d (global), got %d", who, I3D_SH_ESTIMATE, I3D_SH_GLOBAL, l.source);
    if (l.source == I3D_SH_GLOBAL)
    {
        for (int k = 0; k < 9; ++k)
            if (!std::isfinite(l.sh[k])) return fail(e, "%s: sh[%d] is not finite", who, k);
    }
    else if (e->sv_S <= 0 || !e->sv_x)
        return fail(e, "%s: the estimate lighting needs a lighting estimate of the current grid (i3d_estimate_lighting)", who);
    return 0;
}

// The device form of a lighting checked by check_sh_lighting
ShLight sh_light(const I3DEngine* e, const I3DShLighting& l)
{
    ShLight L{};
    L.global = l.source == I3D_SH_GLOBAL ? 1 : 0;
    for (int k = 0; k < 9; ++k) L.sh[k] = l.sh[k];
    if (!L.global) { L.sg = e->sv_grid; L.sub_sh = e->sv_x; L.S = e->sv_S; }
    return L;
}

// The colour pass of a mode other than I3D_MESH_COLOR_VOXEL into e->mesh.vis_rgb; the geometric modes read the sdf the mesh is cut from
void colorize(I3DEngine* e, int32_t sdf_source, int32_t mode)
{
    mesh::colorize(e->mesh, e->timing, e->grid_view(sdf_source == 0 ? e->sdf0.p : e->sdf, e->alb), e->sv_grid, e->sv_x, e->sv_S, mode, e->stream);
}

// The extraction of the surface of prm.sdf_source, coloured by the voxel colours or by a colour mode (validated by the caller)
int extract_mesh(I3DEngine* e, const I3DMeshParams& prm, int32_t color_mode, I3DMeshInfo* info)
{
    if (color_mode != I3D_MESH_COLOR_VOXEL) colorize(e, prm.sdf_source, color_mode);
    MeshGrid g;
    g.n = e->n; g.x = e->x.p; g.y = e->y.p; g.z = e->z.p; g.sdf = prm.sdf_source == 0 ? e->sdf0.p : e->sdf; g.weight = e->weight.p;
    g.rgb = color_mode == I3D_MESH_COLOR_VOXEL ? e->rgb.p : e->mesh.vis_rgb.p;
    g.nbr = e->nbr.p; g.keys = e->up_keys.p; g.vals = e->up_vals.p; g.mask = e->hash_cap - 1; g.voxel_size = e->voxel_size;
    std::string err;
    e->tex.have = false; e->raster.have = false;
    if (mesh::extract(e->mesh, g, prm.largest_component_only != 0, info, err, e->stream)) return fail(e, "%s", err.c_str());
    return 0;
}

// The grid as the renderer marches it, without its voxel box (the render module adds it): the sdf of sdf_source, and the per-voxel SH
// only for photometric outputs
RenderGrid render_grid(const I3DEngine* e, int32_t sdf_source, bool photometric)
{
    RenderGrid rg{};
    rg.g = e->grid_view(sdf_source == 0 ? e->sdf0.p : e->sdf, e->alb);
    if (!photometric) rg.g.sh = nullptr;
    rg.keys = e->up_keys.p; rg.vals = e->up_vals.p; rg.mask = e->hash_cap - 1;
    rg.sh_has = photometric ? e->sh_has.p : nullptr;
    return rg;
}

// Renders frames ids[0..n) (validated by the caller) with the camera of the frame scans: k_pose_mats' float poses and select_cam's
// intrinsics.  Refuses, before it writes anything, intrinsics (after pyr_scale) that are not finite with fx, fy > 0 and distortion that
// is not finite.
int render_keyframes(I3DEngine* e, int32_t n, const int32_t* ids, const I3DRenderParams& P, I3DRenderStats* stats)
{
    cudaStream_t st = e->stream;
    const int F = e->F;
    double hc9[9];
    CK(cudaMemcpyAsync(hc9, e->cam + 6 * static_cast<size_t>(F), 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const SelectCam sc = select_cam(e, hc9, 0.0f);
    if (!(std::isfinite(sc.fx) && sc.fx > 0.0f && std::isfinite(sc.fy) && sc.fy > 0.0f && std::isfinite(sc.cx) && std::isfinite(sc.cy)))
        return fail(e, "i3d_render_keyframes: the camera needs finite intrinsics with fx, fy > 0 (fx %g, fy %g, cx %g, cy %g after pyr_scale %g)",
                    sc.fx, sc.fy, sc.cx, sc.cy, e->pyr_scale);
    for (int k = 0; k < 5; ++k)
        if (!std::isfinite(sc.d[k])) return fail(e, "i3d_render_keyframes: distortion coefficient %d is not finite", k);
    RenderCam cam;
    cam.fx = sc.fx; cam.fy = sc.fy; cam.cx = sc.cx; cam.cy = sc.cy; cam.dist_zero = sc.dist_zero;
    for (int k = 0; k < 5; ++k) cam.d[k] = sc.d[k];
    e->render.rt.ensure(12 * static_cast<size_t>(F));
    k_pose_mats<<<blocks_for(F, 64), 64, 0, st>>>(F, e->cam, e->render.rt.p);
    render::keyframes(e->render, e->timing, render_grid(e, P.sdf_source, P.photometric != 0), cam, e->render.rt.p, n, ids, e->W, e->H, e->depth.p,
                      e->lum.p, P.planes, P.photometric != 0, stats, st);
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
    { const char* v = std::getenv("I3D_PCG_FUSED"); e->pcg_fused = !(v && v[0] == '0'); }
    const int rc = guarded(e, [&]() {
        CK(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
        e->timing.pool.resize(4096);
        for (auto& ev : e->timing.pool) CK(cudaEventCreate(&ev));
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
    for (auto& ev : e->timing.pool) cudaEventDestroy(ev);
    if (e->mesh.ev_ready) for (auto& ev : e->mesh.ev) cudaEventDestroy(ev);
    if (e->tex.ev_ready) for (auto& ev : e->tex.ev) cudaEventDestroy(ev);
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
        e->n = n; e->voxel_size = voxel_size; e->truncation = voxel_size * 5.0f;
        forget_voxel_set(e);
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
        install_frames(e, F, W, H, pyr_scale, [&]() {
            CK(cudaMemcpyAsync(e->lum.p, lum, cnt * sizeof(float), cudaMemcpyHostToDevice, e->stream));
            CK(cudaMemcpyAsync(e->depth.p, depth, cnt * sizeof(float), cudaMemcpyHostToDevice, e->stream));
        });
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
        collect_kernel_times(e->timing, e->stream);
        e->timing.phases["launches"].count = e->launches;
        e->timing.phases["host_syncs"].count = e->host_syncs;
        // the reference's three phase timers (NLSSolver::ProblemInfo::time_add/time_build, SolverInfo::time_solve)
        info->time_add = (e->timing.phases["select"].ms + e->timing.phases["build"].ms) * 1e-3;
        info->time_build = 0.0;
        info->time_solve = e->timing.phases["solve"].ms * 1e-3;
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
        begin_timing(e->timing, {"light_subvolumes", "light_accumulate", "light_solve", "light_interpolate"});
        const GridView g = e->grid_view(e->sdf, e->alb);
        SubvolGrid sg;
        sg.inv_size = 1.0f / P.subvolume_size;
        // ---- Subvolumes::compute ----
        e->sv_scalars.ensure(8);
        {
            Timer t(e->timing, e->stream, "light_subvolumes");
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
            e->sv_grid = sg;
            e->sv_index.ensure(3 * static_cast<size_t>(S)); e->sv_nbr.ensure(6 * static_cast<size_t>(S)); e->sv_deg.ensure(static_cast<size_t>(S));
            k_svsh_indices<<<blocks_for(static_cast<size_t>(cells)), kThreads, 0, st>>>(sg, e->sv_index.p, e->sv_nbr.p, S);
        }
        const int S = e->sv_S;
        const size_t M = 9 * static_cast<size_t>(S);
        // ---- data rows -> per-subvolume normal equations ----
        e->sv_acc.ensure(static_cast<size_t>(S) * kLightAcc);
        {
            Timer t(e->timing, e->stream, "light_accumulate");
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
            Timer t(e->timing, e->stream, "light_solve");
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
            Timer t(e->timing, e->stream, "light_interpolate");
            k_svsh_interpolate<<<blocks_for(n), kThreads, 0, st>>>(g, sg, P.thres_shell, e->sv_x, e->sh.p, e->sh_has.p);
            t.stop();
            e->have_sh = true;
        }
        collect_kernel_times(e->timing, e->stream);
        CK(cudaGetLastError());
        info->time_accumulate = (e->timing.phases["light_subvolumes"].ms + e->timing.phases["light_accumulate"].ms) * 1e-3;
        info->time_solve = e->timing.phases["light_solve"].ms * 1e-3;
        info->time_interpolate = e->timing.phases["light_interpolate"].ms * 1e-3;
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
        begin_timing(e->timing, {"recolor"});
        double hc9[9];
        CK(cudaMemcpyAsync(hc9, e->cam + 6 * static_cast<size_t>(F), 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        e->Rt.ensure(12 * static_cast<size_t>(F));
        e->recolor_counts.ensure(2);
        CK(cudaMemsetAsync(e->recolor_counts.p, 0, 2 * sizeof(unsigned long long), st));
        {
            Timer t(e->timing, e->stream, "recolor");
            if (pose_world_to_cam) CK(cudaMemcpyAsync(e->Rt.p, pose_world_to_cam, 12 * static_cast<size_t>(F) * sizeof(float), cudaMemcpyHostToDevice, st));
            else k_pose_mats<<<blocks_for(F, 64), 64, 0, st>>>(F, e->cam, e->Rt.p);
            const size_t smem = 12 * static_cast<size_t>(F) * sizeof(float);
            auto kern = (K <= 5) ? k_recolor<5> : k_recolor<I3D_MAX_OBS>;
            if (smem > 48 * 1024) CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
            kern<<<blocks_for(static_cast<size_t>(e->n)), kThreads, smem, st>>>(e->grid_view(e->sdf, e->alb), e->frame_view(), e->color.p, e->Rt.p,
                                                                               select_cam(e, hc9, max_occlusion_distance), cull_view(e, nullptr), K,
                                                                               e->rgb.p, e->recolor_counts.p);
        }
        unsigned long long hcnt[2] = {0, 0};
        CK(cudaMemcpyAsync(hcnt, e->recolor_counts.p, sizeof(hcnt), cudaMemcpyDeviceToHost, st));
        collect_kernel_times(e->timing, e->stream);
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
        begin_timing(e->timing, {"prune"});
        int m = 0;
        {
            Timer t(e->timing, e->stream, "prune");
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
                e->n = 0;
                forget_voxel_set(e);
                collect_kernel_times(e->timing, e->stream);
                if (num_voxels_out) *num_voxels_out = 0;
                return 0;
            }
            if (install_grid(e, m, [&](const VoxelArrays& out) { k_gather_voxels<<<blocks_for(static_cast<size_t>(m)), kThreads, 0, st>>>(m, e->act.p, g, out); }))
                return fail(e, "i3d_clear_voxels_outside_thin_shell: internal error (duplicate voxels)");
        }
        collect_kernel_times(e->timing, e->stream);
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
        begin_timing(e->timing, {"upsample"});
        {
            Timer t(e->timing, e->stream, "upsample");
            const GridView g = e->grid_view(e->sdf, e->alb);
            if (install_grid(e, m, [&](const VoxelArrays& out) { k_upsample<<<blocks_for(static_cast<size_t>(m)), kThreads, 0, st>>>(g, e->up_keys.p, e->up_vals.p, e->hash_cap - 1, out); }))
                return fail(e, "i3d_upsample_grid: internal error (duplicate voxels)");
            // SparseVoxelGrid::create(voxelSize * 0.5f): truncation = 5 * voxel size (src/sparse_voxel_grid.cpp:48)
            e->voxel_size = e->voxel_size * 0.5f; e->truncation = e->voxel_size * 5.0f;
        }
        collect_kernel_times(e->timing, e->stream);
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

// ---- RGB-D fusion (i3d_fusion.cuh) ------------------------------------------------------------
uint64_t i3d_sizeof_fusion_params(void) { return sizeof(I3DFusionParams); }

void i3d_default_fusion_params(I3DFusionParams* p)
{
    std::memset(p, 0, sizeof(*p));
    p->voxel_size = 0.004f; p->depth_min = 0.1f; p->depth_max = 4.0f;
    p->integration_weight_sample = 10.0f;
    p->discont_window_size = 2; p->correct_sdf_iterations = 10;
}

int i3d_fusion_begin(I3DEngine* e, const I3DFusionParams* params)
{
    if (!e || !params) return 1;
    e->fusion.active = false;
    if (e->world > 1) return fail(e, "i3d_fusion_begin: fusion runs on one GPU (world = %d)", e->world);
    if (!(params->voxel_size > 0.00001f)) return fail(e, "i3d_fusion_begin: voxel_size %g must be > 1e-5 (SparseVoxelGrid::create)", params->voxel_size);
    if (params->correct_sdf_iterations < 0 || params->discont_window_size < 0 || params->initial_capacity < 0)
        return fail(e, "i3d_fusion_begin: negative correct_sdf_iterations, discont_window_size or initial_capacity");
    return guarded(e, [&]() {
        fusion::begin(e->fusion, e->timing, *params, e->stream);
        e->fusion.active = true;
        return 0;
    });
}

int i3d_fusion_integrate(I3DEngine* e, int32_t F, const I3DFusionCamera* depth_cam, const float* depth, const I3DFusionCamera* color_cam,
                         const uint8_t* bgr, const float* pose_cam_to_world, const float* pose_world_to_cam)
{
    if (!e) return 1;
    if (!e->fusion.active) return fail(e, "i3d_fusion_integrate: no fusion in progress (call i3d_fusion_begin first)");
    if (F < 0 || !depth_cam || !color_cam || (F > 0 && (!depth || !bgr || !pose_cam_to_world || !pose_world_to_cam)))
        return fail(e, "i3d_fusion_integrate: bad arguments");
    if (depth_cam->width <= 0 || depth_cam->height <= 0 || color_cam->width <= 0 || color_cam->height <= 0)
        return fail(e, "i3d_fusion_integrate: bad camera dimensions");
    const int rc = guarded(e, [&]() {
        std::string err;
        if (fusion::integrate_host(e->fusion, e->timing, F, *depth_cam, depth, *color_cam, bgr, pose_cam_to_world, pose_world_to_cam, err, e->stream))
            return fail(e, "i3d_fusion_integrate: %s", err.c_str());
        return 0;
    });
    if (rc != 0) e->fusion.active = false;
    return rc;
}

// ---- the sensor store: the raw sequence on the device (DESIGN.md §6l) -------------------------------
int i3d_sensor_frames_begin(I3DEngine* e, const I3DFusionCamera* depth_cam, const I3DFusionCamera* color_cam, int32_t capacity)
{
    if (!e) return 1;
    if (!pinhole_ok(depth_cam) || !pinhole_ok(color_cam))
        return fail(e, "i3d_sensor_frames_begin: bad camera (a positive size, finite intrinsics and fx, fy > 0 are needed)");
    if (capacity <= 0) return fail(e, "i3d_sensor_frames_begin: capacity must be > 0 (got %d)", capacity);
    e->sensor.F = 0; e->sensor.cap = 0;
    e->fusion.ref_id = -1;             // the _ref odometry's reference is a frame of the store being replaced (DESIGN.md §6q)
    return guarded(e, [&]() { frames::sensor_begin(e->sensor, *depth_cam, *color_cam, capacity); return 0; });
}

int i3d_sensor_frames_add(I3DEngine* e, int32_t F, const float* depth, const uint8_t* bgr)
{
    if (!e) return 1;
    if (e->sensor.cap <= 0) return fail(e, "i3d_sensor_frames_add: no sensor store (call i3d_sensor_frames_begin first)");
    if (F <= 0 || !depth || !bgr) return fail(e, "i3d_sensor_frames_add: need F > 0 frames and non-NULL buffers (F = %d)", F);
    if (F > e->sensor.cap - e->sensor.F)
        return fail(e, "i3d_sensor_frames_add: %d more frames exceed the capacity of %d (%d stored)", F, e->sensor.cap, e->sensor.F);
    return guarded(e, [&]() { frames::sensor_add(e->sensor, F, depth, bgr, e->stream); return 0; });
}

int32_t i3d_sensor_num_frames(const I3DEngine* e) { return e ? e->sensor.F : 0; }

int i3d_sensor_keyframe_scores(I3DEngine* e, double* scores)
{
    if (!e) return 1;
    if (e->sensor.F <= 0) return fail(e, "i3d_sensor_keyframe_scores: no frames in the sensor store");
    if (!scores) return fail(e, "i3d_sensor_keyframe_scores: scores is NULL");
    const int W = e->sensor.ccam.width, H = e->sensor.ccam.height;
    if (W < 5 || H < 5) return fail(e, "i3d_sensor_keyframe_scores: frames of %d x %d px; the 9-tap blur filter needs at least 5 px on each axis", W, H);
    return guarded(e, [&]() { frames::sensor_keyframe_scores(e->scores, e->timing, e->sensor, scores, e->stream); return 0; });
}

// Checks n > 0 and every id against the store; the message names `who`
static int check_sensor_ids(I3DEngine* e, const char* who, int32_t n, const int32_t* ids)
{
    if (e->sensor.F <= 0) return fail(e, "%s: no frames in the sensor store", who);
    if (n <= 0 || !ids) return fail(e, "%s: need n > 0 frame ids (n = %d)", who, n);
    for (int32_t k = 0; k < n; ++k)
        if (ids[k] < 0 || ids[k] >= e->sensor.F) return fail(e, "%s: frame id %d (entry %d) is out of range [0, %d)", who, ids[k], k, e->sensor.F);
    return 0;
}

int i3d_fusion_integrate_sensor(I3DEngine* e, int32_t n, const int32_t* ids, const float* pose_cam_to_world, const float* pose_world_to_cam)
{
    if (!e) return 1;
    if (!e->fusion.active) return fail(e, "i3d_fusion_integrate_sensor: no fusion in progress (call i3d_fusion_begin first)");
    if (check_sensor_ids(e, "i3d_fusion_integrate_sensor", n, ids)) return 1;
    if (!pose_cam_to_world || !pose_world_to_cam) return fail(e, "i3d_fusion_integrate_sensor: poses must not be NULL");
    const int rc = guarded(e, [&]() {
        const SensorStore& ss = e->sensor;
        std::string err;
        if (fusion::integrate(e->fusion, e->timing, n, ss.dcam, ss.depth.p, ss.ccam, ss.bgr.p, ids, pose_cam_to_world, pose_world_to_cam, err, e->stream))
            return fail(e, "i3d_fusion_integrate_sensor: %s", err.c_str());
        return 0;
    });
    if (rc != 0) e->fusion.active = false;
    return rc;
}

int i3d_select_rgbd_frames(I3DEngine* e, int32_t n, const int32_t* ids)
{
    if (!e) return 1;
    if (check_sensor_ids(e, "i3d_select_rgbd_frames", n, ids)) return 1;
    e->rgbd.F = 0;
    return guarded(e, [&]() { frames::select(e->rgbd, e->timing, e->sensor, n, ids, e->stream); return 0; });
}

int i3d_fusion_finish(I3DEngine* e, int64_t* num_voxels_out)
{
    if (!e) return 1;
    if (!e->fusion.active) return fail(e, "i3d_fusion_finish: no fusion in progress (call i3d_fusion_begin first)");
    e->fusion.active = false;
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        begin_timing(e->timing, {});                 // the fusion phases were reset by i3d_fusion_begin
        fusion::correct(e->fusion, e->timing, st);
        int m = 0;
        {
            Timer t(e->timing, e->stream, "fusion_finish");
            m = fusion::sort(e->fusion, true, st);
            if (m > 0)
            {
                if (install_grid(e, m, [&](const VoxelArrays& out) { fusion::convert(e->fusion, m, out, st); }))
                    return fail(e, "i3d_fusion_finish: internal error (duplicate voxels)");
                e->voxel_size = e->fusion.p.voxel_size; e->truncation = e->fusion.p.voxel_size * 5.0f;
            }
            else
            {
                // clearInvalidVoxels left nothing: an empty grid, as after a pruning that removes everything
                e->n = 0;
                forget_voxel_set(e);
            }
        }
        collect_kernel_times(e->timing, e->stream);
        e->fusion.n = 0;
        if (num_voxels_out) *num_voxels_out = m;
        return 0;
    });
}

// ---- surface extraction (i3d_mesh.cuh, DESIGN.md §6j) ----------------------------------------------
uint64_t i3d_sizeof_mesh_info(void) { return sizeof(I3DMeshInfo); }

int i3d_extract_mesh(I3DEngine* e, const I3DMeshParams* params, I3DMeshInfo* info)
{
    if (!e) return 1;
    if (!params) return fail(e, "i3d_extract_mesh: params is NULL");
    if (e->n <= 0) return fail(e, "i3d_extract_mesh: no grid");
    if (check_sdf_source(e, "i3d_extract_mesh", params->sdf_source)) return 1;
    return guarded(e, [&]() { return extract_mesh(e, *params, I3D_MESH_COLOR_VOXEL, info); });
}

int i3d_extract_mesh_colored(I3DEngine* e, const I3DMeshParams* params, int32_t color_mode, I3DMeshInfo* info)
{
    if (!e) return 1;
    if (!params) return fail(e, "i3d_extract_mesh_colored: params is NULL");
    if (e->n <= 0) return fail(e, "i3d_extract_mesh_colored: no grid");
    if (check_sdf_source(e, "i3d_extract_mesh_colored", params->sdf_source)) return 1;
    if (check_color_mode(e, "i3d_extract_mesh_colored", color_mode)) return 1;
    return guarded(e, [&]() { return extract_mesh(e, *params, color_mode, info); });
}

int i3d_mode_colors(I3DEngine* e, int32_t sdf_source, int32_t color_mode, uint8_t* rgb)
{
    if (!e) return 1;
    if (e->n <= 0) return fail(e, "i3d_mode_colors: no grid");
    if (!rgb) return fail(e, "i3d_mode_colors: rgb is NULL");
    if (check_sdf_source(e, "i3d_mode_colors", sdf_source)) return 1;
    if (check_color_mode(e, "i3d_mode_colors", color_mode)) return 1;
    return guarded(e, [&]() {
        const uchar4* src = e->rgb.p;
        if (color_mode != I3D_MESH_COLOR_VOXEL) { colorize(e, sdf_source, color_mode); src = e->mesh.vis_rgb.p; }
        e->up_rgb.ensure(3 * static_cast<size_t>(e->n));
        k_interleave_rgb<<<blocks_for(e->n), kThreads, 0, e->stream>>>(e->n, src, e->up_rgb.p);
        CK(cudaMemcpyAsync(rgb, e->up_rgb.p, 3 * static_cast<size_t>(e->n), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        CK(cudaGetLastError());
        return 0;
    });
}

int i3d_download_mesh(I3DEngine* e, float* xyz, uint8_t* rgb, int32_t* faces)
{
    if (!e) return 1;
    if (!e->mesh.have_mesh) return fail(e, "i3d_download_mesh: no mesh (call i3d_extract_mesh after the last change of the voxel set)");
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t V = static_cast<size_t>(e->mesh.mesh_V), F = static_cast<size_t>(e->mesh.mesh_F);
        if (xyz && V) CK(cudaMemcpyAsync(xyz, e->mesh.mesh_vpos, 3 * V * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (rgb && V) CK(cudaMemcpyAsync(rgb, e->mesh.mesh_vcol, 3 * V, cudaMemcpyDeviceToHost, st));
        if (faces && F) CK(cudaMemcpyAsync(faces, e->mesh.mesh_faces, F * sizeof(int3), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    });
}

// ---- simplifying the resident mesh (i3d_mesh.cuh, DESIGN.md §6s) ------------------------------------
uint64_t i3d_sizeof_simplify_params(void) { return sizeof(I3DSimplifyParams); }
uint64_t i3d_sizeof_simplify_info(void) { return sizeof(I3DSimplifyInfo); }

int i3d_simplify_mesh(I3DEngine* e, const I3DSimplifyParams* params, I3DSimplifyInfo* info)
{
    if (!e) return 1;
    if (!params) return fail(e, "i3d_simplify_mesh: params is NULL");
    if (!e->mesh.have_mesh) return fail(e, "i3d_simplify_mesh: no mesh (call i3d_extract_mesh after the last change of the voxel set)");
    const float cell = params->cell_size;
    if (!std::isfinite(cell) || !(cell > 0.0f)) return fail(e, "i3d_simplify_mesh: cell_size must be finite and > 0, got %g", static_cast<double>(cell));
    return guarded(e, [&]() {
        std::string err;
        if (mesh::simplify(e->mesh, cell, info, err, e->stream)) return fail(e, "%s", err.c_str());
        e->tex.have = false; e->raster.have = false;
        return 0;
    });
}

// ---- baking the keyframes' colour into a texture atlas of the resident mesh (i3d_texture.cuh, DESIGN.md §6t) ------------
uint64_t i3d_sizeof_texture_params(void) { return sizeof(I3DTextureParams); }
uint64_t i3d_sizeof_texture_info(void) { return sizeof(I3DTextureInfo); }

void i3d_default_texture_params(I3DTextureParams* p)
{
    std::memset(p, 0, sizeof(*p));
    p->texels_per_face = 12; p->max_occlusion_distance = 0.02f; p->max_num_observations = 5;
}

int i3d_bake_texture(I3DEngine* e, const I3DTextureParams* params, const float* pose_world_to_cam, I3DTextureInfo* info)
{
    static const char* who = "i3d_bake_texture";
    if (!e) return 1;
    if (!params) return fail(e, "%s: params is NULL", who);
    if (e->world > 1) return fail(e, "%s: the bake runs on one GPU (world = %d)", who, e->world);
    if (!e->mesh.have_mesh) return fail(e, "%s: no mesh (call i3d_extract_mesh after the last change of the voxel set)", who);
    if (e->mesh.mesh_F <= 0) return fail(e, "%s: the resident mesh has no faces", who);
    if (e->F <= 0 || !e->have_cam) return fail(e, "%s: frames and camera must be uploaded first", who);
    if (!e->have_color) return fail(e, "%s: no colour frames of the current frame size (i3d_upload_color_frames)", who);
    const int S = params->texels_per_face, K = params->max_num_observations;
    if (S < I3D_TEXTURE_MIN_TEXELS_PER_FACE || S > I3D_TEXTURE_MAX_TEXELS_PER_FACE)
        return fail(e, "%s: texels_per_face must be in [%d, %d], got %d", who, I3D_TEXTURE_MIN_TEXELS_PER_FACE, I3D_TEXTURE_MAX_TEXELS_PER_FACE, S);
    if (K < 0 || K > I3D_MAX_OBS) return fail(e, "%s: max_num_observations must be in [0, %d], got %d", who, I3D_MAX_OBS, K);
    if (!std::isfinite(params->max_occlusion_distance)) return fail(e, "%s: max_occlusion_distance must be finite", who);
    TexLayout L;
    if (!texture::layout(e->mesh.mesh_F, S, L))
        return fail(e, "%s: %lld faces at %d texels per face need an atlas side above I3D_TEXTURE_MAX_SIDE (%d)", who,
                    static_cast<long long>(e->mesh.mesh_F), S, I3D_TEXTURE_MAX_SIDE);
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const int F = e->F;
        double hc9[9];
        CK(cudaMemcpyAsync(hc9, e->cam + 6 * static_cast<size_t>(F), 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        e->tex.rt.ensure(12 * static_cast<size_t>(F));
        if (pose_world_to_cam) CK(cudaMemcpyAsync(e->tex.rt.p, pose_world_to_cam, 12 * static_cast<size_t>(F) * sizeof(float), cudaMemcpyHostToDevice, st));
        else k_pose_mats<<<blocks_for(F, 64), 64, 0, st>>>(F, e->cam, e->tex.rt.p);
        const TexMesh m{static_cast<int32_t>(e->mesh.mesh_F), e->mesh.mesh_vpos, e->mesh.mesh_vcol, e->mesh.mesh_faces};
        texture::bake(e->tex, e->timing, m, L, e->frame_view(), e->color.p, select_cam(e, hc9, params->max_occlusion_distance), cull_view(e, nullptr), K, info, st);
        return 0;
    });
}

int i3d_download_texture(I3DEngine* e, uint8_t* rgb, float* uv)
{
    if (!e) return 1;
    if (!e->tex.have) return fail(e, "i3d_download_texture: no texture (call i3d_bake_texture after the last extraction or simplification of the mesh)");
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        if (rgb) CK(cudaMemcpyAsync(rgb, e->tex.rgb.p, 3 * static_cast<size_t>(e->tex.W) * e->tex.H, cudaMemcpyDeviceToHost, st));
        if (uv) CK(cudaMemcpyAsync(uv, e->tex.uv.p, 6 * static_cast<size_t>(e->tex.F) * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    });
}

// ---- albedo and shading of the baked texture, and relighting (i3d_texture.cuh, i3d_raster.cuh, DESIGN.md §6x) ----------
uint64_t i3d_sizeof_sh_lighting(void) { return sizeof(I3DShLighting); }
uint64_t i3d_sizeof_intrinsic_texture_params(void) { return sizeof(I3DIntrinsicTextureParams); }
uint64_t i3d_sizeof_intrinsic_texture_info(void) { return sizeof(I3DIntrinsicTextureInfo); }

void i3d_default_sh_lighting(I3DShLighting* p)
{
    std::memset(p, 0, sizeof(*p));
    p->source = I3D_SH_ESTIMATE;
}

void i3d_default_intrinsic_texture_params(I3DIntrinsicTextureParams* p)
{
    std::memset(p, 0, sizeof(*p));
    i3d_default_sh_lighting(&p->lighting);
    p->min_shading = 0.05f;
}

int i3d_decompose_texture(I3DEngine* e, const I3DIntrinsicTextureParams* params, I3DIntrinsicTextureInfo* info)
{
    static const char* who = "i3d_decompose_texture";
    if (!e) return 1;
    if (!params) return fail(e, "%s: params is NULL", who);
    if (e->world > 1) return fail(e, "%s: the decomposition runs on one GPU (world = %d)", who, e->world);
    if (!e->tex.have) return fail(e, "%s: no texture of the resident mesh (call i3d_bake_texture after the last extraction or simplification)", who);
    if (check_sh_lighting(e, who, params->lighting)) return 1;
    if (!std::isfinite(params->min_shading) || params->min_shading < 0.0f)
        return fail(e, "%s: min_shading must be finite and >= 0, got %g", who, static_cast<double>(params->min_shading));
    return guarded(e, [&]() {
        const TexMesh m{static_cast<int32_t>(e->mesh.mesh_F), e->mesh.mesh_vpos, e->mesh.mesh_vcol, e->mesh.mesh_faces};
        texture::decompose(e->tex, m, sh_light(e, params->lighting), params->min_shading, info, e->stream);
        return 0;
    });
}

int i3d_download_intrinsic_texture(I3DEngine* e, float* albedo, float* shading)
{
    if (!e) return 1;
    if (!(e->tex.have && e->tex.intrinsic))
        return fail(e, "i3d_download_intrinsic_texture: no decomposition of the resident mesh's texture (call i3d_decompose_texture after the last bake)");
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t texels = static_cast<size_t>(e->tex.W) * e->tex.H;
        if (albedo) CK(cudaMemcpyAsync(albedo, e->tex.albedo.p, 3 * texels * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (shading) CK(cudaMemcpyAsync(shading, e->tex.shading.p, texels * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    });
}

int i3d_set_relight(I3DEngine* e, const I3DShLighting* lighting)
{
    static const char* who = "i3d_set_relight";
    if (!e) return 1;
    if (!lighting) return fail(e, "%s: lighting is NULL", who);
    if (lighting->source != I3D_SH_ESTIMATE && lighting->source != I3D_SH_GLOBAL)
        return fail(e, "%s: source must be %d (estimate) or %d (global), got %d", who, I3D_SH_ESTIMATE, I3D_SH_GLOBAL, lighting->source);
    if (lighting->source == I3D_SH_GLOBAL)
        for (int k = 0; k < 9; ++k)
            if (!std::isfinite(lighting->sh[k])) return fail(e, "%s: sh[%d] is not finite", who, k);
    e->relight = *lighting;
    return 0;
}

// ---- distance from the resident mesh to a reference mesh (i3d_distance.cuh, DESIGN.md §6u) -----------
uint64_t i3d_sizeof_distance_params(void) { return sizeof(I3DDistanceParams); }
uint64_t i3d_sizeof_distance_info(void) { return sizeof(I3DDistanceInfo); }

void i3d_default_distance_params(I3DDistanceParams* p)
{
    std::memset(p, 0, sizeof(*p));
    p->samples_per_edge = 2; p->max_distance = 0.01f; p->cell_size = 0.0f;
    p->num_thresholds = 3; p->thresholds[0] = 0.0002f; p->thresholds[1] = 0.0005f; p->thresholds[2] = 0.001f;
}

int i3d_upload_reference_mesh(I3DEngine* e, int64_t V, const float* xyz, int64_t F, const int32_t* faces)
{
    if (!e) return 1;
    return guarded(e, [&]() {
        std::string err;
        if (distance::upload_reference(e->dist, V, xyz, F, faces, err, e->stream)) return fail(e, "i3d_upload_reference_mesh: %s", err.c_str());
        return 0;
    });
}

int i3d_surface_distance(I3DEngine* e, const I3DDistanceParams* params, I3DDistanceInfo* info)
{
    static const char* who = "i3d_surface_distance";
    if (!e) return 1;
    if (!params) return fail(e, "%s: params is NULL", who);
    if (e->world > 1) return fail(e, "%s: the distance runs on one GPU (world = %d)", who, e->world);
    if (!e->mesh.have_mesh) return fail(e, "%s: no mesh (call i3d_extract_mesh after the last change of the voxel set)", who);
    if (e->mesh.mesh_F <= 0) return fail(e, "%s: the resident mesh has no faces", who);
    if (!e->dist.have_ref) return fail(e, "%s: no reference mesh (i3d_upload_reference_mesh)", who);
    const I3DDistanceParams& p = *params;
    if (p.samples_per_edge < 1 || p.samples_per_edge > I3D_DISTANCE_MAX_SAMPLES_PER_EDGE)
        return fail(e, "%s: samples_per_edge must be in [1, %d], got %d", who, I3D_DISTANCE_MAX_SAMPLES_PER_EDGE, p.samples_per_edge);
    if (!std::isfinite(p.max_distance) || !(p.max_distance > 0.0f)) return fail(e, "%s: max_distance must be finite and > 0, got %g", who, static_cast<double>(p.max_distance));
    if (!std::isfinite(p.cell_size) || p.cell_size < 0.0f) return fail(e, "%s: cell_size must be finite and >= 0, got %g", who, static_cast<double>(p.cell_size));
    if (p.num_thresholds < 0 || p.num_thresholds > I3D_DISTANCE_MAX_THRESHOLDS)
        return fail(e, "%s: num_thresholds must be in [0, %d], got %d", who, I3D_DISTANCE_MAX_THRESHOLDS, p.num_thresholds);
    for (int k = 0; k < p.num_thresholds; ++k)
    {
        const float t = p.thresholds[k];
        if (!std::isfinite(t) || t < 0.0f || t > p.max_distance || (k > 0 && t < p.thresholds[k - 1]))
            return fail(e, "%s: thresholds must be finite, ascending and in [0, max_distance]; threshold %d is %g", who, k, static_cast<double>(t));
    }
    return guarded(e, [&]() {
        std::string err;
        const DistMesh a{e->mesh.mesh_V, e->mesh.mesh_F, e->mesh.mesh_vpos, e->mesh.mesh_faces};
        if (distance::compute(e->dist, a, p, info, err, e->stream)) return fail(e, "%s: %s", who, err.c_str());
        return 0;
    });
}

int i3d_download_surface_distance(I3DEngine* e, float* vertex_distance, int32_t* vertex_face)
{
    if (!e) return 1;
    if (!e->dist.have_result) return fail(e, "i3d_download_surface_distance: no result (call i3d_surface_distance first)");
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t V = static_cast<size_t>(e->dist.result_V);
        if (vertex_distance && V) CK(cudaMemcpyAsync(vertex_distance, e->dist.vdist.p, V * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (vertex_face && V) CK(cudaMemcpyAsync(vertex_face, e->dist.vface.p, V * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    });
}

int i3d_debug_set_keep_distance_samples(I3DEngine* e, int on)
{
    if (!e) return 1;
    e->dist.keep = on != 0;
    return 0;
}

int i3d_debug_get_distance_samples(I3DEngine* e, int direction, float* d2, int32_t* face)
{
    if (!e) return 1;
    if (direction < 0 || direction > 1) return fail(e, "i3d_debug_get_distance_samples: direction must be 0 or 1, got %d", direction);
    if (!e->dist.have_keep) return fail(e, "i3d_debug_get_distance_samples: the last i3d_surface_distance kept no samples");
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t n = static_cast<size_t>(e->dist.keep_n[direction]);
        if (d2 && n) CK(cudaMemcpyAsync(d2, e->dist.keep_d2[direction].p, n * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (face && n) CK(cudaMemcpyAsync(face, e->dist.keep_face[direction].p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    });
}

// ---- the voxel grid from a triangle mesh (i3d_grid_from_mesh.cuh, DESIGN.md §6v) -----------------------
uint64_t i3d_sizeof_grid_from_mesh_params(void) { return sizeof(I3DGridFromMeshParams); }
uint64_t i3d_sizeof_grid_from_mesh_info(void) { return sizeof(I3DGridFromMeshInfo); }

void i3d_default_grid_from_mesh_params(I3DGridFromMeshParams* p)
{
    std::memset(p, 0, sizeof(*p));
    p->source = I3D_GRID_FROM_MESH_REFERENCE; p->voxel_size = 0.002f; p->band = 3.0f; p->cell_size = 0.0f;
}

int i3d_grid_from_mesh(I3DEngine* e, const I3DGridFromMeshParams* params, I3DGridFromMeshInfo* info)
{
    static const char* who = "i3d_grid_from_mesh";
    if (!e) return 1;
    if (!params) return fail(e, "%s: params is NULL", who);
    if (e->world > 1) return fail(e, "%s: the conversion runs on one GPU (world = %d)", who, e->world);
    const I3DGridFromMeshParams& p = *params;
    DistMesh m{};
    if (p.source == I3D_GRID_FROM_MESH_REFERENCE)
    {
        if (!e->dist.have_ref) return fail(e, "%s: no reference mesh (i3d_upload_reference_mesh)", who);
        m = DistMesh{e->dist.ref_V, e->dist.ref_F, e->dist.ref_vpos.p, e->dist.ref_faces.p};
    }
    else if (p.source == I3D_GRID_FROM_MESH_RESIDENT)
    {
        if (!e->mesh.have_mesh) return fail(e, "%s: no resident mesh (call i3d_extract_mesh after the last change of the voxel set)", who);
        m = DistMesh{e->mesh.mesh_V, e->mesh.mesh_F, e->mesh.mesh_vpos, e->mesh.mesh_faces};
    }
    else return fail(e, "%s: source must be %d (reference) or %d (resident), got %d", who, I3D_GRID_FROM_MESH_REFERENCE, I3D_GRID_FROM_MESH_RESIDENT, p.source);
    if (m.F <= 0) return fail(e, "%s: the source mesh has no faces", who);
    if (!std::isfinite(p.voxel_size) || !(p.voxel_size > 0.0f)) return fail(e, "%s: voxel_size must be finite and > 0, got %g", who, static_cast<double>(p.voxel_size));
    if (!(p.band > 0.0f && p.band <= I3D_GRID_FROM_MESH_MAX_BAND))
        return fail(e, "%s: band must be in (0, %g] voxels, got %g", who, static_cast<double>(I3D_GRID_FROM_MESH_MAX_BAND), static_cast<double>(p.band));
    if (!std::isfinite(p.cell_size) || p.cell_size < 0.0f) return fail(e, "%s: cell_size must be finite and >= 0, got %g", who, static_cast<double>(p.cell_size));
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        I3DGridFromMeshInfo inf;
        std::string err;
        if (gfm::query(e->gfm, m, p, inf, err, st)) return fail(e, "%s: %s", who, err.c_str());
        const int64_t nc = inf.num_candidate_voxels;
        int mk = 0;
        if (nc > 0)
        {
            const int nscan = static_cast<int>((nc + kScanChunk - 1) / kScanChunk);
            e->scan_counts.ensure(static_cast<size_t>(nscan) + 1); e->scan_total.ensure(1); e->act.ensure(static_cast<size_t>(nc));
            k_scan_count<<<nscan, kThreads, 0, st>>>(nc, e->gfm.keep.p, 1, e->scan_counts.p);
            k_scan_blocks<<<1, 1024, 0, st>>>(nscan, e->scan_counts.p, e->scan_total.p);
            k_scan_scatter<<<nscan, kThreads, 0, st>>>(nc, e->gfm.keep.p, 1, e->scan_counts.p, e->act.p);
            CK(cudaMemcpyAsync(&mk, e->scan_total.p, sizeof(int), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            CK(cudaGetLastError());
        }
        if (mk <= 0) return fail(e, "%s: no voxel lies within the band of a face (%lld candidates)", who, static_cast<long long>(nc));
        cudaEvent_t ev[2];
        CK(cudaEventCreate(&ev[0])); CK(cudaEventCreate(&ev[1]));
        CK(cudaEventRecord(ev[0], st));
        const int hdup = install_grid(e, mk, [&](const VoxelArrays& out) { gfm::gather(e->gfm, e->act.p, mk, out, st); });
        CK(cudaEventRecord(ev[1], st));
        CK(cudaEventSynchronize(ev[1]));
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, ev[0], ev[1]));
        CK(cudaEventDestroy(ev[0])); CK(cudaEventDestroy(ev[1]));
        if (hdup) return fail(e, "%s: internal error (duplicate voxels)", who);
        e->voxel_size = p.voxel_size; e->truncation = p.voxel_size * 5.0f;
        inf.ms_install = ms;
        if (info) *info = inf;
        return 0;
    });
}

int i3d_debug_get_grid_from_mesh_voxels(I3DEngine* e, int32_t* face, int8_t* feature)
{
    if (!e) return 1;
    if (!e->gfm.have_last) return fail(e, "i3d_debug_get_grid_from_mesh_voxels: no conversion (call i3d_grid_from_mesh first)");
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t n = static_cast<size_t>(e->gfm.last_n);
        if (face) CK(cudaMemcpyAsync(face, e->gfm.last_face.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (feature) CK(cudaMemcpyAsync(feature, e->gfm.last_feat.p, n, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    });
}

// ---- rendering the surface into the keyframes (i3d_render.cuh, DESIGN.md §6m) ----------------------
uint64_t i3d_sizeof_render_params(void) { return sizeof(I3DRenderParams); }
uint64_t i3d_sizeof_render_stats(void) { return sizeof(I3DRenderStats); }

void i3d_default_render_params(I3DRenderParams* p)
{
    std::memset(p, 0, sizeof(*p));
    p->sdf_source = 1; p->planes = I3D_RENDER_ALL; p->photometric = 1;
}

int i3d_render_keyframes(I3DEngine* e, int32_t n, const int32_t* ids, const I3DRenderParams* params, I3DRenderStats* stats)
{
    static const char* who = "i3d_render_keyframes";
    if (!e) return 1;
    if (!params) return fail(e, "%s: params is NULL", who);
    if (e->world > 1) return fail(e, "%s: rendering runs on one GPU (world = %d)", who, e->world);
    if (e->n <= 0) return fail(e, "%s: no grid", who);
    if (e->F <= 0) return fail(e, "%s: no frames", who);
    if (!e->have_cam) return fail(e, "%s: camera not set", who);
    if (n <= 0 || !ids) return fail(e, "%s: need n > 0 frame ids (n = %d)", who, n);
    if (n > kRenderMaxViews) return fail(e, "%s: %d views exceed the %d of one call", who, n, kRenderMaxViews);
    for (int32_t k = 0; k < n; ++k)
        if (ids[k] < 0 || ids[k] >= e->F) return fail(e, "%s: frame id %d (entry %d) is out of range [0, %d)", who, ids[k], k, e->F);
    if (check_sdf_source(e, who, params->sdf_source)) return 1;
    if (params->planes < 0 || params->planes > I3D_RENDER_ALL) return fail(e, "%s: planes must be a mask in [0, %d], got %d", who, I3D_RENDER_ALL, params->planes);
    if (params->photometric != 0 && params->photometric != 1) return fail(e, "%s: photometric must be 0 or 1, got %d", who, params->photometric);
    if ((params->planes & (I3D_RENDER_SHADING | I3D_RENDER_INTENSITY)) && !params->photometric)
        return fail(e, "%s: the shading and intensity planes need photometric = 1", who);
    if (params->photometric && !e->have_sh)
        return fail(e, "%s: shading, intensity and photometric pairs need the per-voxel SH of the current grid (i3d_set_sh or i3d_estimate_lighting)", who);
    return guarded(e, [&]() { return render_keyframes(e, n, ids, *params, stats); });
}

int i3d_download_render(I3DEngine* e, float* depth, float* normal, float* albedo, float* shading, float* intensity)
{
    if (!e) return 1;
    if (!e->render.have_render) return fail(e, "i3d_download_render: no render (call i3d_render_keyframes after the last change of the grid or frames)");
    const struct { float* dst; int bit; const char* name; } want[5] = {{depth, I3D_RENDER_DEPTH, "depth"}, {normal, I3D_RENDER_NORMAL, "normal"},
        {albedo, I3D_RENDER_ALBEDO, "albedo"}, {shading, I3D_RENDER_SHADING, "shading"}, {intensity, I3D_RENDER_INTENSITY, "intensity"}};
    for (const auto& w : want)
        if (w.dst && !(e->render.planes & w.bit)) return fail(e, "i3d_download_render: the %s plane was not rendered", w.name);
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t img = static_cast<size_t>(e->render.n) * e->W * e->H * sizeof(float);
        if (depth) CK(cudaMemcpyAsync(depth, e->render.depth.p, img, cudaMemcpyDeviceToHost, st));
        if (normal) CK(cudaMemcpyAsync(normal, e->render.normal.p, 3 * img, cudaMemcpyDeviceToHost, st));
        if (albedo) CK(cudaMemcpyAsync(albedo, e->render.albedo.p, img, cudaMemcpyDeviceToHost, st));
        if (shading) CK(cudaMemcpyAsync(shading, e->render.shading.p, img, cudaMemcpyDeviceToHost, st));
        if (intensity) CK(cudaMemcpyAsync(intensity, e->render.intensity.p, img, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    });
}

int i3d_debug_set_render_skip(I3DEngine* e, int on)
{
    if (!e) return 1;
    e->render.skip = on != 0;
    return 0;
}

// ---- rasterizing the resident mesh into the keyframes and into new views (i3d_raster.cuh, DESIGN.md §6w) ----------------
uint64_t i3d_sizeof_raster_params(void) { return sizeof(I3DRasterParams); }
uint64_t i3d_sizeof_raster_camera(void) { return sizeof(I3DRasterCamera); }
uint64_t i3d_sizeof_raster_stats(void) { return sizeof(I3DRasterStats); }
uint64_t i3d_sizeof_raster_info(void) { return sizeof(I3DRasterInfo); }

void i3d_default_raster_params(I3DRasterParams* p)
{
    std::memset(p, 0, sizeof(*p));
    p->planes = I3D_RASTER_ALL; p->color_source = I3D_RASTER_COLOR_VERTEX;
}

// The refusals both raster calls share
static int check_raster_call(I3DEngine* e, const char* who, int32_t n, const I3DRasterParams* params)
{
    if (!params) return fail(e, "%s: params is NULL", who);
    if (e->world > 1) return fail(e, "%s: rasterization runs on one GPU (world = %d)", who, e->world);
    if (!e->mesh.have_mesh) return fail(e, "%s: no mesh (call i3d_extract_mesh after the last change of the voxel set)", who);
    if (e->mesh.mesh_F <= 0) return fail(e, "%s: the resident mesh has no faces", who);
    if (n <= 0) return fail(e, "%s: need n > 0 views (n = %d)", who, n);
    if (n > kRenderMaxViews) return fail(e, "%s: %d views exceed the %d of one call", who, n, kRenderMaxViews);
    if (params->planes < 0 || params->planes > I3D_RASTER_ALL) return fail(e, "%s: planes must be a mask in [0, %d], got %d", who, I3D_RASTER_ALL, params->planes);
    const int cs = params->color_source;
    if (cs != I3D_RASTER_COLOR_NONE && cs != I3D_RASTER_COLOR_VERTEX && cs != I3D_RASTER_COLOR_TEXTURE && cs != I3D_RASTER_COLOR_RELIT)
        return fail(e, "%s: color_source must be %d (none), %d (vertex), %d (texture) or %d (relit), got %d", who, I3D_RASTER_COLOR_NONE,
                    I3D_RASTER_COLOR_VERTEX, I3D_RASTER_COLOR_TEXTURE, I3D_RASTER_COLOR_RELIT, cs);
    if (cs == I3D_RASTER_COLOR_TEXTURE && !e->tex.have)
        return fail(e, "%s: the texture colour source needs a texture of the resident mesh (i3d_bake_texture after the last extraction or simplification)", who);
    if (cs == I3D_RASTER_COLOR_RELIT && !(e->tex.have && e->tex.intrinsic))
        return fail(e, "%s: the relit colour source needs a decomposition of the resident mesh's texture (i3d_decompose_texture after the last bake)", who);
    if (cs == I3D_RASTER_COLOR_RELIT && check_sh_lighting(e, who, e->relight)) return 1;
    return 0;
}

// A camera the rasterizer can use: finite intrinsics with fx, fy > 0 and finite distortion
static int check_raster_camera(I3DEngine* e, const char* who, const RenderCam& c)
{
    if (!(std::isfinite(c.fx) && c.fx > 0.0f && std::isfinite(c.fy) && c.fy > 0.0f && std::isfinite(c.cx) && std::isfinite(c.cy)))
        return fail(e, "%s: the camera needs finite intrinsics with fx, fy > 0 (fx %g, fy %g, cx %g, cy %g)", who, c.fx, c.fy, c.cx, c.cy);
    for (int k = 0; k < 5; ++k)
        if (!std::isfinite(c.d[k])) return fail(e, "%s: distortion coefficient %d is not finite", who, k);
    return 0;
}

static RastMesh raster_mesh(const I3DEngine* e, int color_source)
{
    RastMesh m{static_cast<int32_t>(e->mesh.mesh_F), e->mesh.mesh_vpos, e->mesh.mesh_vcol, e->mesh.mesh_faces, nullptr, 0, 0, 0, 0};
    if (color_source == I3D_RASTER_COLOR_TEXTURE || color_source == I3D_RASTER_COLOR_RELIT)
    {
        m.tex_rgb = e->tex.rgb.p; m.tex_W = e->tex.W; m.tex_H = e->tex.H; m.tex_S = e->tex.S; m.tex_cols = e->tex.cols;
    }
    return m;
}

// The relit source's inputs of a call (validated by check_raster_call)
static void raster_relight(const I3DEngine* e, int color_source, RastCall& c)
{
    if (color_source != I3D_RASTER_COLOR_RELIT) return;
    c.albedo = e->tex.albedo.p;
    c.light = sh_light(e, e->relight);
}

int i3d_rasterize_keyframes(I3DEngine* e, int32_t n, const int32_t* ids, const I3DRasterParams* params, I3DRasterStats* stats, I3DRasterInfo* info)
{
    static const char* who = "i3d_rasterize_keyframes";
    if (!e) return 1;
    if (check_raster_call(e, who, n, params)) return 1;
    if (!ids) return fail(e, "%s: ids is NULL", who);
    if (e->F <= 0 || !e->have_cam) return fail(e, "%s: frames and camera must be uploaded first", who);
    for (int32_t k = 0; k < n; ++k)
        if (ids[k] < 0 || ids[k] >= e->F) return fail(e, "%s: frame id %d (entry %d) is out of range [0, %d)", who, ids[k], k, e->F);
    if (params->color_source != I3D_RASTER_COLOR_NONE && !e->have_color)
        return fail(e, "%s: a colour source needs colour frames of the current frame size (i3d_upload_color_frames)", who);
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const int F = e->F;
        double hc9[9];
        CK(cudaMemcpyAsync(hc9, e->cam + 6 * static_cast<size_t>(F), 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        const SelectCam sc = select_cam(e, hc9, 0.0f);
        RenderCam cam;
        cam.fx = sc.fx; cam.fy = sc.fy; cam.cx = sc.cx; cam.cy = sc.cy; cam.dist_zero = sc.dist_zero;
        for (int k = 0; k < 5; ++k) cam.d[k] = sc.d[k];
        if (check_raster_camera(e, who, cam)) return 1;
        e->raster.rt.ensure(12 * static_cast<size_t>(F));
        k_pose_mats<<<blocks_for(F, 64), 64, 0, st>>>(F, e->cam, e->raster.rt.p);
        RastCall c{n, e->W, e->H, ids, e->raster.rt.p, e->depth.p, params->color_source != I3D_RASTER_COLOR_NONE ? e->color.p : nullptr,
                   params->planes, params->color_source, true};
        raster_relight(e, params->color_source, c);
        raster::run(e->raster, e->timing, raster_mesh(e, params->color_source), cam, c, stats, info, st);
        return 0;
    });
}

int i3d_rasterize_views(I3DEngine* e, int32_t n, const I3DRasterCamera* camera, const float* pose_world_to_cam, const I3DRasterParams* params,
                        I3DRasterInfo* info)
{
    static const char* who = "i3d_rasterize_views";
    if (!e) return 1;
    if (check_raster_call(e, who, n, params)) return 1;
    if (!camera) return fail(e, "%s: camera is NULL", who);
    if (!pose_world_to_cam) return fail(e, "%s: pose_world_to_cam is NULL", who);
    if (camera->width < 1 || camera->width > I3D_RASTER_MAX_SIDE || camera->height < 1 || camera->height > I3D_RASTER_MAX_SIDE)
        return fail(e, "%s: width and height must be in [1, %d], got %d x %d", who, I3D_RASTER_MAX_SIDE, camera->width, camera->height);
    RenderCam cam;
    cam.fx = camera->fx; cam.fy = camera->fy; cam.cx = camera->cx; cam.cy = camera->cy; cam.dist_zero = 1;
    for (int k = 0; k < 5; ++k) { cam.d[k] = camera->distortion[k]; if (cam.d[k] != 0.0f) cam.dist_zero = 0; }
    if (check_raster_camera(e, who, cam)) return 1;
    for (int64_t k = 0; k < 12 * static_cast<int64_t>(n); ++k)
        if (!std::isfinite(pose_world_to_cam[k])) return fail(e, "%s: pose entry %lld (view %lld) is not finite", who, static_cast<long long>(k), static_cast<long long>(k / 12));
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        e->raster.rt.ensure(12 * static_cast<size_t>(n));
        CK(cudaMemcpyAsync(e->raster.rt.p, pose_world_to_cam, 12 * static_cast<size_t>(n) * sizeof(float), cudaMemcpyHostToDevice, st));
        RastCall c{n, camera->width, camera->height, nullptr, e->raster.rt.p, nullptr, nullptr, params->planes, params->color_source, false};
        raster_relight(e, params->color_source, c);
        raster::run(e->raster, e->timing, raster_mesh(e, params->color_source), cam, c, nullptr, info, st);
        return 0;
    });
}

int i3d_download_raster(I3DEngine* e, float* depth, int32_t* face, float* bary, float* normal, uint8_t* rgb)
{
    static const char* who = "i3d_download_raster";
    if (!e) return 1;
    if (!e->raster.have) return fail(e, "%s: no rasterization of the resident mesh (call i3d_rasterize_keyframes or i3d_rasterize_views)", who);
    const struct { const void* dst; int bit; const char* name; } want[5] = {{depth, I3D_RASTER_DEPTH, "depth"}, {face, I3D_RASTER_FACE, "face"},
        {bary, I3D_RASTER_BARY, "bary"}, {normal, I3D_RASTER_NORMAL, "normal"}, {rgb, I3D_RASTER_RGB, "rgb"}};
    for (const auto& w : want)
        if (w.dst && !(e->raster.planes & w.bit)) return fail(e, "%s: the %s plane was not rendered", who, w.name);
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t img = static_cast<size_t>(e->raster.n) * e->raster.W * e->raster.H;
        if (depth) CK(cudaMemcpyAsync(depth, e->raster.depth.p, img * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (face) CK(cudaMemcpyAsync(face, e->raster.face.p, img * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (bary) CK(cudaMemcpyAsync(bary, e->raster.bary.p, 2 * img * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (normal) CK(cudaMemcpyAsync(normal, e->raster.normal.p, 3 * img * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (rgb) CK(cudaMemcpyAsync(rgb, e->raster.rgb.p, 3 * img, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    });
}

int i3d_debug_set_raster_binning(I3DEngine* e, int on)
{
    if (!e) return 1;
    e->raster.binning = on != 0;
    return 0;
}

int i3d_debug_set_raster_batch(I3DEngine* e, int views)
{
    if (!e) return 1;
    if (views < 0) return fail(e, "i3d_debug_set_raster_batch: views must be >= 0, got %d", views);
    e->raster.max_batch = views;
    return 0;
}

// ---- tracking sensor frames against the surface (i3d_track.cuh, DESIGN.md §6n) -------------------
uint64_t i3d_sizeof_track_params(void) { return sizeof(I3DTrackParams); }
uint64_t i3d_sizeof_track_info(void) { return sizeof(I3DTrackInfo); }

void i3d_default_track_params(I3DTrackParams* p)
{
    std::memset(p, 0, sizeof(*p));
    p->sdf_source = 0; p->num_levels = 3;
    p->iterations[0] = 10; p->iterations[1] = 5; p->iterations[2] = 4; p->iterations[3] = 0;
    p->max_distance = 0.05f; p->min_normal_cos = static_cast<float>(std::cos(20.0 * M_PI / 180.0));
    p->min_correspondences = 100;
}

// The refusals of a call that tracks frames side by side: n <= 65535 and distinct ids
static int check_track_batch(I3DEngine* e, const char* who, int32_t n, const int32_t* ids)
{
    if (n > kRenderMaxViews) return fail(e, "%s: %d frames exceed the %d of one call", who, n, kRenderMaxViews);
    std::vector<uint8_t> seen(e->sensor.F, 0);
    for (int32_t k = 0; k < n; ++k)
    {
        if (seen[ids[k]]) return fail(e, "%s: frame id %d is repeated (entry %d); each frame has one pose", who, ids[k], k);
        seen[ids[k]] = 1;
    }
    return 0;
}

// The tracking parameters other than sdf_source; fills the pyramid sizes Wl / Hl
static int check_track_params(I3DEngine* e, const char* who, const I3DTrackParams& P, int* Wl, int* Hl)
{
    if (P.num_levels < 1 || P.num_levels > kTrackMaxLevels) return fail(e, "%s: num_levels must be in 1..%d, got %d", who, kTrackMaxLevels, P.num_levels);
    Wl[0] = e->sensor.dcam.width; Hl[0] = e->sensor.dcam.height;
    for (int l = 1; l < P.num_levels; ++l)
    {
        if (Wl[l - 1] < 3 || Hl[l - 1] < 3)
            return fail(e, "%s: level %d would be built from a %d x %d level; downsampling needs at least 3 px on each axis", who, l, Wl[l - 1], Hl[l - 1]);
        Wl[l] = Wl[l - 1] / 2; Hl[l] = Hl[l - 1] / 2;
    }
    for (int l = 0; l < kTrackMaxLevels; ++l)
        if (P.iterations[l] < 0) return fail(e, "%s: iterations[%d] = %d is negative", who, l, P.iterations[l]);
    if (!(std::isfinite(P.max_distance) && P.max_distance > 0.0f)) return fail(e, "%s: max_distance must be finite and > 0, got %g", who, P.max_distance);
    if (!(P.min_normal_cos >= -1.0f && P.min_normal_cos <= 1.0f)) return fail(e, "%s: min_normal_cos must be in [-1, 1], got %g", who, P.min_normal_cos);
    if (P.min_correspondences < 6) return fail(e, "%s: min_correspondences must be >= 6, got %d", who, P.min_correspondences);
    return 0;
}

static int check_finite_poses(I3DEngine* e, const char* who, int32_t n, const double* pose, const char* what)
{
    for (int64_t i = 0; i < 12 * static_cast<int64_t>(n); ++i)
        if (!std::isfinite(pose[i])) return fail(e, "%s: %s of entry %d is not finite", who, what, static_cast<int>(i / 12));
    return 0;
}

// The refusals of a photometric term (DESIGN.md §6p) and of its local normalisation (§6r, reference: a _ref call); fills col
static int check_track_color(I3DEngine* e, const char* who, const I3DTrackColorParams* cp, I3DTrackColorInfo* ci, bool reference, TrackColor& col)
{
    if (!cp) return fail(e, "%s: color params must not be NULL", who);
    for (int l = 0; l < kTrackMaxLevels; ++l)
        if (!(std::isfinite(cp->weight[l]) && cp->weight[l] >= 0.0f)) return fail(e, "%s: weight[%d] must be finite and >= 0, got %g", who, l, cp->weight[l]);
    if (!(std::isfinite(cp->max_color_diff) && cp->max_color_diff > 0.0f))
        return fail(e, "%s: max_color_diff must be finite and > 0, got %g", who, cp->max_color_diff);
    if (!(std::isfinite(cp->min_color_gradient) && cp->min_color_gradient >= 0.0f))
        return fail(e, "%s: min_color_gradient must be finite and >= 0, got %g", who, cp->min_color_gradient);
    if (cp->norm_radius != 0 && !reference)
        return fail(e, "%s: norm_radius must be 0 with the voxel model, whose model plane is not an image (the _ref calls take it), got %d", who,
                    cp->norm_radius);
    if (cp->norm_radius < 0 || cp->norm_radius > I3D_TRACK_MAX_NORM_RADIUS)
        return fail(e, "%s: norm_radius must be in 0..%d, got %d", who, I3D_TRACK_MAX_NORM_RADIUS, cp->norm_radius);
    if (cp->norm_radius > 0 && !(std::isfinite(cp->norm_eps) && cp->norm_eps > 0.0f))
        return fail(e, "%s: norm_eps must be finite and > 0 with norm_radius > 0, got %g", who, cp->norm_eps);
    col = TrackColor{cp, &e->sensor, ci};
    return 0;
}

// The references of a _ref call (DESIGN.md §6q), n frames; completes col
struct TrackReference { bool on; const int32_t* ids; const double* pose; };
static int check_track_reference(I3DEngine* e, const char* who, int32_t n, const TrackReference& ref, TrackColor& col)
{
    if (!ref.ids || !ref.pose) return fail(e, "%s: ref_ids and ref_pose must not be NULL", who);
    for (int32_t k = 0; k < n; ++k)
        if (ref.ids[k] < 0 || ref.ids[k] >= e->sensor.F)
            return fail(e, "%s: reference id %d (entry %d) is out of range (%d stored frames)", who, ref.ids[k], k, e->sensor.F);
    if (check_finite_poses(e, who, n, ref.pose, "the reference pose")) return 1;
    col.ref_ids = ref.ids; col.ref_pose = ref.pose;
    return 0;
}
static constexpr TrackReference kNoReference{false, nullptr, nullptr};

// i3d_track_sensor_frames, with the photometric term cp when it is not nullptr (the _rgbd call) and its reference model (the _ref call)
static int track_sensor_frames(I3DEngine* e, const char* who, int32_t n, const int32_t* ids, const double* pose_in, const I3DTrackParams* params,
                               double* pose_out, I3DTrackInfo* info, bool rgbd, const I3DTrackColorParams* cp, I3DTrackColorInfo* ci,
                               const TrackReference& ref = kNoReference)
{
    if (!e) return 1;
    if (!params || !pose_in || !pose_out) return fail(e, "%s: params, pose_in and pose_out must not be NULL", who);
    if (e->world > 1) return fail(e, "%s: tracking runs on one GPU (world = %d)", who, e->world);
    if (e->n <= 0) return fail(e, "%s: no grid", who);
    if (check_sensor_ids(e, who, n, ids)) return 1;
    if (check_track_batch(e, who, n, ids)) return 1;
    if (check_finite_poses(e, who, n, pose_in, "the input pose")) return 1;
    const I3DTrackParams& P = *params;
    if (check_sdf_source(e, who, P.sdf_source)) return 1;
    int Wl[kTrackMaxLevels], Hl[kTrackMaxLevels];
    if (check_track_params(e, who, P, Wl, Hl)) return 1;
    TrackColor col{};
    if (rgbd && check_track_color(e, who, cp, ci, ref.on, col)) return 1;
    if (ref.on && check_track_reference(e, who, n, ref, col)) return 1;
    return guarded(e, [&]() {
        track::sensor_frames(e->track, e->render, e->timing, render_grid(e, P.sdf_source, false), e->sensor.dcam, e->sensor.depth.p, e->sensor.F, n, ids, pose_in, P,
                             Wl, Hl, pose_out, info, e->stream, rgbd ? &col : nullptr);
        return 0;
    });
}

int i3d_track_sensor_frames(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const I3DTrackParams* params, double* pose_out,
                            I3DTrackInfo* info)
{
    return track_sensor_frames(e, "i3d_track_sensor_frames", n, ids, pose_in, params, pose_out, info, false, nullptr, nullptr);
}

int i3d_track_sensor_frames_rgbd(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const I3DTrackParams* params,
                                 const I3DTrackColorParams* color, double* pose_out, I3DTrackInfo* info, I3DTrackColorInfo* color_info)
{
    return track_sensor_frames(e, "i3d_track_sensor_frames_rgbd", n, ids, pose_in, params, pose_out, info, true, color, color_info);
}

int i3d_track_sensor_frames_rgbd_ref(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const int32_t* ref_ids, const double* ref_pose,
                                     const I3DTrackParams* params, const I3DTrackColorParams* color, double* pose_out, I3DTrackInfo* info,
                                     I3DTrackColorInfo* color_info)
{
    return track_sensor_frames(e, "i3d_track_sensor_frames_rgbd_ref", n, ids, pose_in, params, pose_out, info, true, color, color_info,
                               TrackReference{true, ref_ids, ref_pose});
}

// The checks of the two calls that track against the fusion in progress, up to the poses
static int check_fusion_track(I3DEngine* e, const char* who, int32_t n, const int32_t* ids, const I3DTrackParams* params, double* pose_out)
{
    if (!params || !pose_out) return fail(e, "%s: params and pose_out must not be NULL", who);
    if (e->world > 1) return fail(e, "%s: tracking runs on one GPU (world = %d)", who, e->world);
    if (!e->fusion.active) return fail(e, "%s: no fusion in progress (call i3d_fusion_begin first)", who);
    return check_sensor_ids(e, who, n, ids);
}

static int fusion_track_sensor_frames(I3DEngine* e, const char* who, int32_t n, const int32_t* ids, const double* pose_in,
                                      const I3DTrackParams* params, double* pose_out, I3DTrackInfo* info, bool rgbd, const I3DTrackColorParams* cp,
                                      I3DTrackColorInfo* ci, const TrackReference& ref = kNoReference)
{
    if (!e) return 1;
    if (!pose_in) return fail(e, "%s: pose_in must not be NULL", who);
    if (check_fusion_track(e, who, n, ids, params, pose_out)) return 1;
    if (check_track_batch(e, who, n, ids)) return 1;
    if (check_finite_poses(e, who, n, pose_in, "the input pose")) return 1;
    const I3DTrackParams& P = *params;
    if (P.sdf_source != 0) return fail(e, "%s: sdf_source must be 0 (the fusion volume holds one sdf), got %d", who, P.sdf_source);
    int Wl[kTrackMaxLevels], Hl[kTrackMaxLevels];
    if (check_track_params(e, who, P, Wl, Hl)) return 1;
    TrackColor col{};
    if (rgbd && check_track_color(e, who, cp, ci, ref.on, col)) return 1;
    if (ref.on && check_track_reference(e, who, n, ref, col)) return 1;
    return guarded(e, [&]() {
        if (track::fusion_frames(e->track, e->fusion, e->render.skip, e->timing, e->sensor, n, ids, pose_in, P, Wl, Hl, pose_out, info, e->stream,
                                 rgbd ? &col : nullptr))
            return fail(e, "%s: the fusion volume has no voxel with weight > 0", who);
        return 0;
    });
}

int i3d_fusion_track_sensor_frames(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const I3DTrackParams* params, double* pose_out,
                                   I3DTrackInfo* info)
{
    return fusion_track_sensor_frames(e, "i3d_fusion_track_sensor_frames", n, ids, pose_in, params, pose_out, info, false, nullptr, nullptr);
}

int i3d_fusion_track_sensor_frames_rgbd(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const I3DTrackParams* params,
                                        const I3DTrackColorParams* color, double* pose_out, I3DTrackInfo* info, I3DTrackColorInfo* color_info)
{
    return fusion_track_sensor_frames(e, "i3d_fusion_track_sensor_frames_rgbd", n, ids, pose_in, params, pose_out, info, true, color, color_info);
}

int i3d_fusion_track_sensor_frames_rgbd_ref(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const int32_t* ref_ids,
                                            const double* ref_pose, const I3DTrackParams* params, const I3DTrackColorParams* color, double* pose_out,
                                            I3DTrackInfo* info, I3DTrackColorInfo* color_info)
{
    return fusion_track_sensor_frames(e, "i3d_fusion_track_sensor_frames_rgbd_ref", n, ids, pose_in, params, pose_out, info, true, color, color_info,
                                      TrackReference{true, ref_ids, ref_pose});
}

// reference: the loop's own reference model (DESIGN.md §6q)
static int fusion_track_and_integrate_sensor(I3DEngine* e, const char* who, int32_t n, const int32_t* ids, const double* pose_first,
                                             const I3DTrackParams* params, double* pose_out, I3DTrackInfo* info, bool rgbd,
                                             const I3DTrackColorParams* cp, I3DTrackColorInfo* ci, bool reference = false)
{
    if (!e) return 1;
    if (check_fusion_track(e, who, n, ids, params, pose_out)) return 1;
    if (pose_first ? check_finite_poses(e, who, 1, pose_first, "pose_first") : 0) return 1;
    if (!pose_first && e->fusion.motion == 0)
        return fail(e, "%s: pose_first is NULL and the fusion has no motion state (a fusion begun or integrated since the last odometry call)", who);
    const I3DTrackParams& P = *params;
    if (P.sdf_source != 0) return fail(e, "%s: sdf_source must be 0 (the fusion volume holds one sdf), got %d", who, P.sdf_source);
    int Wl[kTrackMaxLevels], Hl[kTrackMaxLevels];
    if (check_track_params(e, who, P, Wl, Hl)) return 1;
    TrackColor col{};
    if (rgbd && check_track_color(e, who, cp, ci, reference, col)) return 1;
    const int rc = guarded(e, [&]() {
        std::string err;
        if (track::odometry(e->track, e->fusion, e->render.skip, e->timing, e->sensor, n, ids, pose_first, P, Wl, Hl, pose_out, info, err, e->stream,
                            rgbd ? &col : nullptr, reference))
            return fail(e, "%s: %s", who, err.c_str());
        return 0;
    });
    if (rc != 0) e->fusion.active = false;
    return rc;
}

int i3d_fusion_track_and_integrate_sensor(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_first, const I3DTrackParams* params,
                                          double* pose_out, I3DTrackInfo* info)
{
    return fusion_track_and_integrate_sensor(e, "i3d_fusion_track_and_integrate_sensor", n, ids, pose_first, params, pose_out, info, false, nullptr,
                                             nullptr);
}

int i3d_fusion_track_and_integrate_sensor_rgbd(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_first, const I3DTrackParams* params,
                                               const I3DTrackColorParams* color, double* pose_out, I3DTrackInfo* info, I3DTrackColorInfo* color_info)
{
    return fusion_track_and_integrate_sensor(e, "i3d_fusion_track_and_integrate_sensor_rgbd", n, ids, pose_first, params, pose_out, info, true, color,
                                             color_info);
}

int i3d_fusion_track_and_integrate_sensor_rgbd_ref(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_first, const I3DTrackParams* params,
                                                   const I3DTrackColorParams* color, double* pose_out, I3DTrackInfo* info, I3DTrackColorInfo* color_info)
{
    return fusion_track_and_integrate_sensor(e, "i3d_fusion_track_and_integrate_sensor_rgbd_ref", n, ids, pose_first, params, pose_out, info, true,
                                             color, color_info, true);
}

int i3d_debug_get_track_system(I3DEngine* e, double* sums, double* pose_cam_to_world)
{
    if (!e) return 1;
    if (e->track.n <= 0) return fail(e, "i3d_debug_get_track_system: no tracking call");
    return guarded(e, [&]() {
        const int n = e->track.n;
        if (sums) CK(cudaMemcpyAsync(sums, e->track.sys.p, static_cast<size_t>(n) * kTrackVals * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
        std::vector<TrackState> hs(pose_cam_to_world ? n : 0);
        if (pose_cam_to_world) CK(cudaMemcpyAsync(hs.data(), e->track.state.p, n * sizeof(TrackState), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        for (size_t k = 0; k < hs.size(); ++k) std::memcpy(pose_cam_to_world + 12 * k, hs[k].T, 12 * sizeof(double));
        return 0;
    });
}

int i3d_debug_get_track_planes(I3DEngine* e, int32_t level, float* depth, float* normal, float* pred_depth, float* pred_normal, uint8_t* mask,
                               int32_t* frames)
{
    if (!e) return 1;
    if (e->track.n <= 0) return fail(e, "i3d_debug_get_track_planes: no tracking call");
    if (level < 0 || level >= e->track.levels) return fail(e, "i3d_debug_get_track_planes: level %d was not built (%d levels)", level, e->track.levels);
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t m = static_cast<size_t>(e->track.last_m);
        const size_t lv = m * e->track.W[level] * e->track.H[level], img = m * e->track.W[0] * e->track.H[0];
        if (depth) CK(cudaMemcpyAsync(depth, e->track.depth[level].p, lv * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (normal) CK(cudaMemcpyAsync(normal, e->track.nrm[level].p, 3 * lv * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (pred_depth) CK(cudaMemcpyAsync(pred_depth, e->track.pdepth.p, img * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (pred_normal) CK(cudaMemcpyAsync(pred_normal, e->track.pnrm.p, 3 * img * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (mask) CK(cudaMemcpyAsync(mask, e->track.mask.p, img, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (frames) *frames = static_cast<int32_t>(m);
        return 0;
    });
}

// ---- the photometric term of tracking (i3d_track.cuh, DESIGN.md §6p) ------------------------------
uint64_t i3d_sizeof_track_color_params(void) { return sizeof(I3DTrackColorParams); }
uint64_t i3d_sizeof_track_color_info(void) { return sizeof(I3DTrackColorInfo); }

void i3d_default_track_color_params(I3DTrackColorParams* p)
{
    std::memset(p, 0, sizeof(*p));
    for (int l = 0; l < kTrackMaxLevels; ++l) p->weight[l] = 0.05f;      // measured on C2 (DESIGN.md §6p)
    p->max_color_diff = 0.1f; p->min_color_gradient = 0.01f;
}

int i3d_debug_get_track_color_planes(I3DEngine* e, int32_t level, float* model_intensity, float* intensity, float* grad_x, float* grad_y,
                                     int32_t* frames)
{
    static const char* who = "i3d_debug_get_track_color_planes";
    if (!e) return 1;
    if (e->track.n <= 0 || !e->track.color) return fail(e, "%s: the last tracking call had no photometric term", who);
    if (level < 0 || level >= e->track.levels) return fail(e, "%s: level %d was not built (%d levels)", who, level, e->track.levels);
    if (model_intensity && e->track.reference)
        return fail(e, "%s: the last call took its model from reference frames (i3d_debug_get_track_reference_planes)", who);
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const size_t m = static_cast<size_t>(e->track.last_m);
        const size_t lv = m * e->track.W[level] * e->track.H[level], img = m * e->track.W[0] * e->track.H[0];
        if (model_intensity) CK(cudaMemcpyAsync(model_intensity, e->track.pint.p, img * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (intensity) CK(cudaMemcpyAsync(intensity, e->track.inten[level].p, lv * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (grad_x) CK(cudaMemcpyAsync(grad_x, e->track.gx[level].p, lv * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (grad_y) CK(cudaMemcpyAsync(grad_y, e->track.gy[level].p, lv * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (frames) *frames = static_cast<int32_t>(m);
        return 0;
    });
}

int i3d_debug_get_track_color_system(I3DEngine* e, double* sums)
{
    if (!e) return 1;
    if (e->track.n <= 0 || !e->track.color) return fail(e, "i3d_debug_get_track_color_system: the last tracking call had no photometric term");
    return guarded(e, [&]() {
        if (sums)
            CK(cudaMemcpyAsync(sums, e->track.sys_c.p, static_cast<size_t>(e->track.n) * kTrackVals * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        return 0;
    });
}

// ---- the reference model of the photometric term (i3d_track.cuh, DESIGN.md §6q) --------------------
void i3d_default_track_color_ref_params(I3DTrackColorParams* p)
{
    i3d_default_track_color_params(p);
    for (int l = 0; l < kTrackMaxLevels; ++l) p->weight[l] = 0.01f;      // measured on C2 (DESIGN.md §6q)
}

void i3d_default_track_color_lni_params(I3DTrackColorParams* p)
{
    i3d_default_track_color_ref_params(p);
    for (int l = 0; l < kTrackMaxLevels; ++l) p->weight[l] = 0.005f;      // measured on C2 (DESIGN.md §6r)
    p->max_color_diff = 1.0f; p->min_color_gradient = 0.05f;
    p->norm_radius = 3; p->norm_eps = 0.01f;
}

int i3d_debug_get_track_reference_planes(I3DEngine* e, int32_t level, float* model, float* ref_intensity, float* ref_depth, int32_t* frames)
{
    static const char* who = "i3d_debug_get_track_reference_planes";
    if (!e) return 1;
    if (e->track.n <= 0 || !e->track.reference) return fail(e, "%s: the last tracking call had no reference model", who);
    if (level < 0 || level >= e->track.levels) return fail(e, "%s: level %d was not built (%d levels)", who, level, e->track.levels);
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const int m = e->track.last_m, W0 = e->track.W[0], H0 = e->track.H[0], Wl = e->track.W[level], Hl = e->track.H[level];
        const size_t lv = static_cast<size_t>(m) * Wl * Hl;
        if (ref_intensity) CK(cudaMemcpyAsync(ref_intensity, e->track.ref_inten[level].p, lv * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (ref_depth) CK(cudaMemcpyAsync(ref_depth, e->track.ref_depth[level].p, lv * sizeof(float), cudaMemcpyDeviceToHost, st));
        // the model plane is in the level-0 layout: pixel (u, v) of level l at (2^l v) W0 + 2^l u
        std::vector<float> full(model ? static_cast<size_t>(m) * W0 * H0 : 0);
        if (model)
            CK(cudaMemcpyAsync(full.data(), (level == 0 ? e->track.pint : e->track.ref_model[level]).p, full.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        const size_t s = size_t{1} << level;
        for (size_t z = 0; model && z < static_cast<size_t>(m); ++z)
            for (size_t v = 0; v < static_cast<size_t>(Hl); ++v)
                for (size_t u = 0; u < static_cast<size_t>(Wl); ++u)
                    model[(z * Hl + v) * Wl + u] = full[(z * H0 + s * v) * W0 + s * u];
        if (frames) *frames = m;
        return 0;
    });
}

// ---- keyframe selection and the RGB-D pyramid (i3d_frames.cuh, DESIGN.md §6i) --------------------
int i3d_keyframe_scores(I3DEngine* e, int32_t F, int32_t W, int32_t H, const uint8_t* bgr, double* scores)
{
    if (!e) return 1;
    if (F <= 0 || !bgr || !scores) return fail(e, "i3d_keyframe_scores: need F > 0 frames and non-NULL buffers (F = %d)", F);
    if (W < 5 || H < 5) return fail(e, "i3d_keyframe_scores: frames of %d x %d px; the 9-tap blur filter needs at least 5 px on each axis", W, H);
    return guarded(e, [&]() { frames::keyframe_scores(e->scores, e->timing, F, W, H, bgr, scores, e->stream); return 0; });
}

int i3d_upload_rgbd_frames(I3DEngine* e, int32_t F, int32_t W, int32_t H, const uint8_t* bgr, const float* depth, const float* lum)
{
    if (!e) return 1;
    if (F <= 0 || W <= 0 || H <= 0) return fail(e, "i3d_upload_rgbd_frames: bad dimensions (F = %d, %d x %d)", F, W, H);
    if (!bgr || !depth) return fail(e, "i3d_upload_rgbd_frames: bgr and depth must not be NULL");
    e->rgbd.F = 0;
    return guarded(e, [&]() { frames::upload(e->rgbd, F, W, H, bgr, depth, lum, e->stream); return 0; });
}

int i3d_use_rgbd_level(I3DEngine* e, int32_t lvl, int32_t* W_out, int32_t* H_out)
{
    if (!e) return 1;
    if (e->rgbd.F <= 0) return fail(e, "i3d_use_rgbd_level: no frame store (call i3d_upload_rgbd_frames first)");
    if (lvl < 0) return fail(e, "i3d_use_rgbd_level: negative level %d", lvl);
    int W = e->rgbd.W, H = e->rgbd.H;
    for (int k = 1; k <= lvl; ++k)
    {
        if (W < 3 || H < 3)
            return fail(e, "i3d_use_rgbd_level: level %d would be built from a %d x %d level; downsampling needs at least 3 px on each axis", lvl, W, H);
        W /= 2; H /= 2;
    }
    return guarded(e, [&]() {
        cudaStream_t st = e->stream;
        const int F = e->rgbd.F;
        const size_t cnt = static_cast<size_t>(F) * W * H;
        begin_timing(e->timing, {"frames_level"});
        install_frames(e, F, W, H, std::ldexp(1.0, -lvl), [&]() { frames::level(e->rgbd, e->timing, lvl, e->lum.p, e->depth.p, st); });
        if (lvl == 0)
        {
            e->color.ensure(3 * cnt);
            CK(cudaMemcpyAsync(e->color.p, e->rgbd.bgr.p, 3 * cnt, cudaMemcpyDeviceToDevice, st));
            e->have_color = true;
        }
        collect_kernel_times(e->timing, e->stream);
        CK(cudaGetLastError());
        if (W_out) *W_out = W;
        if (H_out) *H_out = H;
        return 0;
    });
}

int i3d_debug_get_frames(I3DEngine* e, float* lum, float* depth, uint8_t* bgr)
{
    if (!e) return 1;
    if (e->F <= 0) return fail(e, "i3d_debug_get_frames: no frames on the device");
    if (bgr && !e->have_color) return fail(e, "i3d_debug_get_frames: no colour frames at the current size");
    return guarded(e, [&]() {
        const size_t cnt = static_cast<size_t>(e->F) * e->W * e->H;
        if (lum) CK(cudaMemcpyAsync(lum, e->lum.p, cnt * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
        if (depth) CK(cudaMemcpyAsync(depth, e->depth.p, cnt * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
        if (bgr) CK(cudaMemcpyAsync(bgr, e->color.p, 3 * cnt, cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
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
    auto it = e->timing.phases.find(name);
    return it == e->timing.phases.end() ? 0.0 : it->second.ms;
}
int64_t i3d_phase_count(const I3DEngine* e, const char* name)
{
    auto it = e->timing.phases.find(name);
    return it == e->timing.phases.end() ? 0 : it->second.count;
}

int64_t i3d_debug_num_slots(const I3DEngine* e) { return e->have_iter ? static_cast<int64_t>(e->K) * e->stride : 0; }
int i3d_debug_set_kernel_timers(I3DEngine* e, int level)
{
    if (!e) return 1;
    e->timing.level = level > 0 ? 1 : 0;
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
        std::vector<float4> jt(jac_colmajor ? EgRows::kTiles * S : 0);
        std::vector<float2> jtail(jac_colmajor ? S : 0);
        if (jac_colmajor)
        {
            CK(cudaMemcpyAsync(jt.data(), e->Jt.p, jt.size() * sizeof(float4), cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(jtail.data(), e->Jtail.p, jtail.size() * sizeof(float2), cudaMemcpyDeviceToHost, st));
        }
        CK(cudaStreamSynchronize(st));
        if (jac_colmajor)
            for (size_t i = 0; i < S; ++i)
            {
                for (int c = 0; c < EgRows::kTiles; ++c)
                {
                    const float4 t = jt[c * S + i];
                    jac_colmajor[(4 * c) * S + i] = t.x; jac_colmajor[(4 * c + 1) * S + i] = t.y;
                    jac_colmajor[(4 * c + 2) * S + i] = t.z; jac_colmajor[(4 * c + 3) * S + i] = t.w;
                }
                jac_colmajor[28 * S + i] = jtail[i].x;
            }
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

int i3d_debug_get_pcg_vectors(I3DEngine* e, float* x, float* p)
{
    if (!e || !e->have_iter) return fail(e, "i3d_debug_get_pcg_vectors: no iteration yet");
    return guarded(e, [&]() {
        const size_t U = static_cast<size_t>(e->U());
        if (x) CK(cudaMemcpyAsync(x, e->v_x.p, U * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
        if (p) CK(cudaMemcpyAsync(p, e->v_p.p, U * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
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
        const int timer_level = e->timing.level;
        const int64_t launches = e->launches;
        e->timing.level = -1;                       // keep the last iteration's kernel table
        GridView g = e->grid_view(e->sdf, e->alb);
        const RegView rv = reg_view(e, e->last_params);
        const EgRows rows = eg_rows(e);
        const SolveVecs sv = solve_vecs(e);
        const Shard sh = e->shard();
        const int64_t hc = e->held_count();
        pdl_launch(e, k_scale_vec, blocks_for(static_cast<size_t>(hc)), kThreads, 0, sv, sh, hc, e->dbg_v.p, 1.0f, sv.ps, e->ctl.p, 0);
        launch_operator(e, g, rv, rows, sv, sh, e->dbg_v.p, 0.0f, 0.0f, 0);
        e->timing.level = timer_level;
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

int64_t i3d_debug_fusion_num_voxels(const I3DEngine* e) { return (e && e->fusion.active) ? e->fusion.n : 0; }

int i3d_debug_get_fusion_volume(I3DEngine* e, int32_t* xyz, float* sdf, float* weight, uint8_t* rgb)
{
    if (!e || !e->fusion.active) return fail(e, "i3d_debug_get_fusion_volume: no fusion in progress");
    return guarded(e, [&]() { fusion::download(e->fusion, xyz, sdf, weight, rgb, e->stream); return 0; });
}

} // extern "C"
