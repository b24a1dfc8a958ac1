/*
 * i3d_kernels.cuh — sm_90a kernels of the joint-refinement engine.
 *
 * Data layout in HBM (all SoA, voxel index = position in the host's iteration order):
 *   grid      x,y,z int32[n]; sdf0, sdf, albedo double[n]; weight float[n]; rgb uchar4[n];
 *             nbr int32[12][n]  (neighbour table: +x,-x,+y,-y,+z,-z,+2x,+2y,+2z,(110),(101),(011); -1 = absent)
 *             sh double[9][n]
 *   frames    lum, depth float[F][H][W]; camera double[6F+9] (poses | intrinsics | distortion)
 *   per GN iteration
 *             flags uint8[n]; act int32[n_a] (compacted active voxels, ascending)
 *             E_g row slots, k-major: slot = k*n_a + a
 *                 J float[29][K*n_a] raw rows (column-major => coalesced for thread-per-voxel access)
 *                 row_frame int32, row_res double (unweighted), row_wraw double, row_w float (final weight)
 *   unknown-space vectors float[U], U = 2n + 6F + 9 : [sdf | albedo | poses | intrinsics | distortion]
 *
 * Reference functions replaced (libintrinsic3d/): see each kernel.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <limits.h>
#include "i3d_math.cuh"
#include "../../include/i3d_types.h"

namespace i3d
{

// neighbour-table slots
enum { NB_XP = 0, NB_XM, NB_YP, NB_YM, NB_ZP, NB_ZM, NB_X2, NB_Y2, NB_Z2, NB_XY, NB_XZ, NB_YZ, NB_COUNT };

// voxel flags
enum : uint8_t { FL_VALID = 1, FL_ACTIVE = 2, FL_RING = 4, FL_FREE_SDF = 8, FL_FREE_ALB = 16, FL_ES_JAC = 32, FL_ROW = 64 /* active and owned by this rank */ };

// Multi-GPU sharding (one process per GPU).  Residual ROWS are owned by the rank that owns their voxel
// (voxel index range [own_begin, own_end) in the host's iteration order); the state and the voxel flags are
// replicated.  Every unknown-space quantity is computed as a partial sum over OWNED rows; unknowns touched by
// rows of more than one rank ("shared", the boundary layers between shards) plus the camera block are summed
// with ONE packed exchange per operator application.
struct Shard
{
    int64_t own_begin, own_end;
    int64_t hv0, hv1;         // index hull of the voxels whose unknowns this rank HOLDS (owned or touched by its rows); [0, n) on one GPU
    int cam_owner;            // this rank adds the camera entries to global reductions
    int defer;                // world > 1: kernels leave PARTIAL sums in their reduce site, the epilogue runs after the allreduce
    int64_t loc_begin, loc_end;   // voxel index range this rank ever reads per-iteration data of (owned + 4 stencil rings); [0, n) on one GPU
    __device__ __forceinline__ bool owns_voxel(int64_t v) const { return v >= own_begin && v < own_end; }
    __device__ __forceinline__ bool owns_unknown(int64_t j, int64_t n) const
    {
        return j < n ? owns_voxel(j) : (j < 2 * n ? owns_voxel(j - n) : cam_owner != 0);
    }
    // number of unknowns the per-unknown kernels of this rank run over: sdf and albedo of the hull + the camera block
    __host__ __device__ __forceinline__ int64_t held_voxel_unknowns() const { return 2 * (hv1 - hv0); }
    // thread index -> unknown index: [sdf of the hull | albedo of the hull | camera].  Pure arithmetic (round 1 went through an index
    // list: one dependent load per access and no 16-byte vector path — k_cg_update was 2x slower on HALF the unknowns at 2 GPUs).
    // Unknowns of the hull that this rank does not hold carry no rows of this rank: their local values are never exchanged or read.
    __device__ __forceinline__ int64_t unknown(int64_t t, int64_t n) const
    {
        const int64_t L = hv1 - hv0;
        return t < L ? hv0 + t : (t < 2 * L ? n + hv0 + (t - L) : 2 * n + (t - 2 * L));
    }
    // four consecutive thread indices starting at e0 (multiple of 4) -> four consecutive, 16-byte aligned unknowns starting at *j0 ?
    __device__ __forceinline__ bool vec4(int64_t e0, int64_t n, int64_t* j0) const
    {
        const int64_t L = hv1 - hv0;
        if (e0 + 4 > 2 * L) return false;
        if (hv0 == 0 && hv1 == n) { *j0 = e0; return true; }      // whole grid: [sdf | albedo] is one contiguous range
        if (e0 < L && e0 + 4 > L) return false;        // would straddle the sdf / albedo boundary
        const int64_t j = e0 < L ? hv0 + e0 : n + hv0 + (e0 - L);
        *j0 = j;
        return (j & 3) == 0;
    }
};

constexpr int kThreads = 256;

// Programmatic dependent launch (sm_90+): the host launches every kernel of the Gauss-Newton iteration with
// cudaLaunchAttributeProgrammaticStreamSerialization (pdl_launch, i3d_engine.cu).  griddepcontrol.wait blocks until the preceding
// grid of the stream has completed and its memory is visible — nothing above it may touch global memory written by a predecessor —
// and griddepcontrol.launch_dependents lets the NEXT grid be scheduled as soon as every CTA of this one has started, so its
// launch latency overlaps this grid's tail.  Without the launch attribute both instructions are no-ops.
__device__ __forceinline__ void pdl_prologue()
{
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

#ifndef I3D_BUILD_MIN_BLOCKS
#define I3D_BUILD_MIN_BLOCKS 2
#endif

struct GridView
{
    int64_t n;
    const int32_t* x; const int32_t* y; const int32_t* z;
    const double* sdf0; const double* sdf; const double* albedo;
    const float* weight;
    const uchar4* rgb;
    const int32_t* nbr;    // [12][n]
    const double* sh;      // [9][n]
    float voxel_size, truncation;
};

struct FrameView
{
    int F, W, H;
    const float* lum; const float* depth;
    double pyr_scale;
};

// ----------------------------------------------------------------------------------------------
// deterministic reductions: block partials -> last block sums them in a fixed order
// ----------------------------------------------------------------------------------------------
struct ReduceSite
{
    double* partials;     // [blocks][NV] (sized by the engine for the largest grid)
    unsigned int* counter;
    double* out;          // [NV]
};

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// returns the block sum in thread 0 (other threads: undefined)
template <class T>
__device__ __forceinline__ T block_sum(T v, T* smem /* >= 32 */)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) smem[wid] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    v = (threadIdx.x < nw) ? smem[threadIdx.x] : T(0);
    if (wid == 0) v = warp_sum(v);
    return v;
}

// Every block calls this with its per-thread values; returns true in ALL threads of the block that
// finished last, after site.out[0..NV) holds the grid totals.
template <int NV>
__device__ __forceinline__ bool grid_reduce(double (&vals)[NV], const ReduceSite& site)
{
    __shared__ double red_smem[32];
    __shared__ bool is_last;
#pragma unroll
    for (int i = 0; i < NV; ++i)
    {
        const double s = block_sum<double>(vals[i], red_smem);
        if (threadIdx.x == 0) site.partials[static_cast<size_t>(blockIdx.x) * NV + i] = s;
    }
    if (threadIdx.x == 0)
    {
        __threadfence();
        const unsigned int ticket = atomicAdd(site.counter, 1u);
        is_last = (ticket == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return false;
    __threadfence();
#pragma unroll
    for (int i = 0; i < NV; ++i)
    {
        double s = 0.0;
        for (unsigned int b = threadIdx.x; b < gridDim.x; b += blockDim.x) s += __ldcg(&site.partials[static_cast<size_t>(b) * NV + i]);
        s = block_sum<double>(s, red_smem);
        if (threadIdx.x == 0) site.out[i] = s;
    }
    if (threadIdx.x == 0) { *site.counter = 0u; __threadfence(); }
    __syncthreads();
    return true;
}

// ----------------------------------------------------------------------------------------------
// warp butterfly reduce-scatter: every lane contributes N values (N multiple of 32); afterwards lane L
// holds, in v[0 .. N/32), the warp-wide sums of the original indices
//     idx(i, L) = i + (N/32)*b0 + (N/16)*b1 + (N/8)*b2 + (N/4)*b3 + (N/2)*b4      (b_k = bit k of L)
// N + log-many shuffles instead of 5N for N independent all-reduces; the results land on distinct lanes,
// so the follow-up atomics of a warp hit distinct addresses (no same-address serialisation).
// ----------------------------------------------------------------------------------------------
template <int HALF, int OFF, int N>
__device__ __forceinline__ void rs_step(float (&v)[N], int lane)
{
    const bool up = (lane & OFF) != 0;
#pragma unroll
    for (int i = 0; i < HALF; ++i)
    {
        const float send = up ? v[i] : v[i + HALF];
        const float keep = up ? v[i + HALF] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
    }
}
template <int N>
__device__ __forceinline__ void warp_reduce_scatter(float (&v)[N], int lane)
{
    static_assert(N % 32 == 0, "N must be a multiple of 32");
    rs_step<N / 2, 16, N>(v, lane);
    rs_step<N / 4, 8, N>(v, lane);
    rs_step<N / 8, 4, N>(v, lane);
    rs_step<N / 16, 2, N>(v, lane);
    rs_step<N / 32, 1, N>(v, lane);
}
template <int N>
__device__ __forceinline__ int rs_index(int i, int lane)
{
    return i + (N / 32) * (lane & 1) + (N / 16) * ((lane >> 1) & 1) + (N / 8) * ((lane >> 2) & 1) + (N / 4) * ((lane >> 3) & 1) + (N / 2) * ((lane >> 4) & 1);
}

// register-array element by run-time index without spilling the array to local memory
__device__ __forceinline__ int fk_select(const int (&fk)[I3D_MAX_OBS], int k)
{
    int r = fk[0];
#pragma unroll
    for (int i = 1; i < I3D_MAX_OBS; ++i) r = (k == i) ? fk[i] : r;
    return r;
}

// ----------------------------------------------------------------------------------------------
// grid upload: hash table + neighbour table (replaces unordered_map::find, sparse_voxel_grid.cpp:166-259)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t pack_key(int x, int y, int z)
{
    return ((static_cast<uint64_t>(x + (1 << 20)) & 0x1FFFFFull) << 42) | ((static_cast<uint64_t>(y + (1 << 20)) & 0x1FFFFFull) << 21) |
           (static_cast<uint64_t>(z + (1 << 20)) & 0x1FFFFFull);
}
__device__ __forceinline__ uint64_t mix64(uint64_t k)
{
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return k;
}
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;

__global__ void k_deinterleave_xyz(int64_t n, const int32_t* __restrict__ xyz, int32_t* __restrict__ x, int32_t* __restrict__ y, int32_t* __restrict__ z,
                                   const uint8_t* __restrict__ rgb3, uchar4* __restrict__ rgb4)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    x[i] = xyz[3 * i]; y[i] = xyz[3 * i + 1]; z[i] = xyz[3 * i + 2];
    rgb4[i] = make_uchar4(rgb3[3 * i], rgb3[3 * i + 1], rgb3[3 * i + 2], 0);
}

__global__ void k_hash_insert(int64_t n, const int32_t* __restrict__ x, const int32_t* __restrict__ y, const int32_t* __restrict__ z,
                              unsigned long long* __restrict__ keys, int32_t* __restrict__ vals, uint64_t mask, int* __restrict__ dup_flag)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    const unsigned long long key = pack_key(x[i], y[i], z[i]);
    uint64_t slot = mix64(key) & mask;
    while (true)
    {
        const unsigned long long prev = atomicCAS(&keys[slot], kEmptyKey, key);
        if (prev == kEmptyKey) { vals[slot] = static_cast<int32_t>(i); return; }
        if (prev == key) { atomicExch(dup_flag, 1); return; }
        slot = (slot + 1) & mask;
    }
}

// (noinline: runs once per grid upload; keeps the 12 probe loops out of the caller)
__device__ __noinline__ int32_t hash_find(const unsigned long long* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask, int x, int y, int z)
{
    const unsigned long long key = pack_key(x, y, z);
    uint64_t slot = mix64(key) & mask;
    while (true)
    {
        const unsigned long long k = keys[slot];
        if (k == key) return vals[slot];
        if (k == kEmptyKey) return -1;
        slot = (slot + 1) & mask;
    }
}

__global__ void k_build_nbr(int64_t n, const int32_t* __restrict__ x, const int32_t* __restrict__ y, const int32_t* __restrict__ z,
                            const unsigned long long* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask, int32_t* __restrict__ nbr)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    const int X = x[i], Y = y[i], Z = z[i];
    const int off[NB_COUNT][3] = {{1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}, {2, 0, 0}, {0, 2, 0}, {0, 0, 2}, {1, 1, 0}, {1, 0, 1}, {0, 1, 1}};
#pragma unroll
    for (int o = 0; o < NB_COUNT; ++o) nbr[static_cast<int64_t>(o) * n + i] = hash_find(keys, vals, mask, X + off[o][0], Y + off[o][1], Z + off[o][2]);
}

__global__ void k_transpose_sh(int64_t n, const double* __restrict__ sh_aos, double* __restrict__ sh_soa)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= 9 * n) return;
    const int64_t v = i / 9; const int k = static_cast<int>(i - 9 * v);
    sh_soa[static_cast<int64_t>(k) * n + v] = sh_aos[i];
}

// ----------------------------------------------------------------------------------------------
// exact float arithmetic (no FMA contraction): must round like oracle.cpp / the reference's float code
// ----------------------------------------------------------------------------------------------
#define FM(a, b) __fmul_rn((a), (b))
#define FA(a, b) __fadd_rn((a), (b))
#define FS(a, b) __fsub_rn((a), (b))
#define FD(a, b) __fdiv_rn((a), (b))

// SDFOperators::computeSurfaceNormal (src/sdf/operators.cpp:58-77): float forward differences.
__device__ __forceinline__ bool surface_normal_f(const GridView& g, int64_t v, float nrm[3])
{
    nrm[0] = nrm[1] = nrm[2] = 0.0f;
    const int32_t ix = g.nbr[NB_XP * g.n + v], iy = g.nbr[NB_YP * g.n + v], iz = g.nbr[NB_ZP * g.n + v];
    if (!(g.weight[v] > 0.0f) || ix < 0 || iy < 0 || iz < 0) return false;
    if (!(g.weight[ix] > 0.0f) || !(g.weight[iy] > 0.0f) || !(g.weight[iz] > 0.0f)) return false;
    const float s0 = static_cast<float>(g.sdf[v]);
    float g0 = FS(static_cast<float>(g.sdf[ix]), s0);
    float g1 = FS(static_cast<float>(g.sdf[iy]), s0);
    float g2 = FS(static_cast<float>(g.sdf[iz]), s0);
    const float sq = FA(FA(FM(g0, g0), FM(g1, g1)), FM(g2, g2));
    const float len = __fsqrt_rn(sq);
    if (len != 0.0f) { g0 = FD(g0, len); g1 = FD(g1, len); g2 = FD(g2, len); }
    nrm[0] = g0; nrm[1] = g1; nrm[2] = g2;
    return !(g0 == 0.0f && g1 == 0.0f && g2 == 0.0f);
}

// Activity and free masks for one GN iteration.
//   active  = Optimizer::addVoxelResiduals' tests (optimizer.cpp:183-193)
//   free    = complement of Optimizer::fixVoxelParams (optimizer.cpp:312-361)
//   ES_JAC  = E_s row has a non-zero derivative (sdf_refined != sdf0; surface_stab_regularizer.h:62-64)
__global__ void k_flags(GridView g, Shard sh, double thres_shell, int fix_all_albedo, uint8_t* __restrict__ flags)
{
    pdl_prologue();
    const int64_t v = sh.loc_begin + blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;      // only the range this rank reads
    if (v >= sh.loc_end) return;
    uint8_t fl = 0;
    const bool valid = g.weight[v] > 0.0f;
    if (valid) fl |= FL_VALID;
    bool ring = true;
#pragma unroll
    for (int o = 0; o < 6; ++o)
    {
        const int32_t nb = g.nbr[static_cast<int64_t>(o) * g.n + v];
        if (nb < 0 || !(g.weight[nb] > 0.0f)) ring = false;
    }
    if (ring) fl |= FL_RING;
    const double s = g.sdf[v];
    const bool inshell = !(fabs(s) > thres_shell);
    if (valid && inshell)
    {
        float nrm[3];
        if (surface_normal_f(g, v, nrm)) { fl |= FL_ACTIVE; if (sh.owns_voxel(v)) fl |= FL_ROW; }
        if (ring) { fl |= FL_FREE_SDF; if (!fix_all_albedo) fl |= FL_FREE_ALB; }
    }
    if ((s - g.sdf0[v]) != 0.0) fl |= FL_ES_JAC;
    flags[v] = fl;
}

// --- stream compaction of active voxels (ascending index) -------------------------------------
constexpr int kScanItems = 8;                         // items per thread
constexpr int kScanChunk = kThreads * kScanItems;     // items per block

__global__ void k_scan_count(int64_t n, const uint8_t* __restrict__ flags, uint8_t bit, int32_t* __restrict__ block_counts)
{
    pdl_prologue();
    __shared__ int smem[32];
    const int64_t base = static_cast<int64_t>(blockIdx.x) * kScanChunk;
    int c = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i)
    {
        const int64_t idx = base + static_cast<int64_t>(i) * kThreads + threadIdx.x;
        if (idx < n && (flags[idx] & bit)) c++;
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
    if (lane == 0) smem[wid] = c;
    __syncthreads();
    if (threadIdx.x == 0)
    {
        int s = 0;
        for (int w = 0; w < kThreads / 32; ++w) s += smem[w];
        block_counts[blockIdx.x] = s;
    }
}

// single block: exclusive scan of block_counts in place; total -> *total
__global__ void k_scan_blocks(int nblocks, int32_t* __restrict__ block_counts, int32_t* __restrict__ total)
{
    pdl_prologue();
    __shared__ int carry;
    __shared__ int wsum[32];
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += blockDim.x)
    {
        const int i = base + threadIdx.x;
        const int v = (i < nblocks) ? block_counts[i] : 0;
        int incl = v;
        const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        if (lane == 31) wsum[wid] = incl;
        __syncthreads();
        if (wid == 0)
        {
            int w = (lane < (blockDim.x >> 5)) ? wsum[lane] : 0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += t; }
            wsum[lane] = w;
        }
        __syncthreads();
        const int woff = (wid > 0) ? wsum[wid - 1] : 0;
        const int excl = carry + woff + incl - v;
        if (i < nblocks) block_counts[i] = excl;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

__global__ void k_scan_scatter(int64_t n, const uint8_t* __restrict__ flags, uint8_t bit, const int32_t* __restrict__ block_offsets,
                               int32_t* __restrict__ out_list, int32_t index_offset = 0)
{
    pdl_prologue();
    __shared__ int wsum[kThreads / 32];
    const int64_t base = static_cast<int64_t>(blockIdx.x) * kScanChunk;
    int running = block_offsets[blockIdx.x];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int i = 0; i < kScanItems; ++i)
    {
        const int64_t idx = base + static_cast<int64_t>(i) * kThreads + threadIdx.x;
        const bool f = idx < n && (flags[idx] & bit);
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        if (lane == 0) wsum[wid] = __popc(bal);
        __syncthreads();
        int woff = 0, tot = 0;
        for (int w = 0; w < kThreads / 32; ++w) { const int c = wsum[w]; if (w < wid) woff += c; tot += c; }
        if (f) out_list[running + woff + __popc(bal & ((1u << lane) - 1u))] = static_cast<int32_t>(idx) + index_offset;
        running += tot;
        __syncthreads();
    }
}

// ----------------------------------------------------------------------------------------------
// k1: observation selection (SDFColorization::collectObservations, src/sdf/colorization.cpp:192-370)
// ----------------------------------------------------------------------------------------------
// math::poseVecAAToMat (src/math.cpp:151-163) in double, cast to float: R[9] row-major, t[3]
__global__ void k_pose_mats(int F, const double* __restrict__ poses, float* __restrict__ Rt /* [F][12] */)
{
    pdl_prologue();
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const double wx = poses[6 * f], wy = poses[6 * f + 1], wz = poses[6 * f + 2];
    const double n2 = wx * wx + wy * wy + wz * wz;
    const double angle = sqrt(n2);
    double ax = wx, ay = wy, az = wz;
    if (n2 > 0.0) { ax = wx / angle; ay = wy / angle; az = wz / angle; }
    const double s = sin(angle), c = cos(angle);
    const double sx = __dmul_rn(s, ax), sy = __dmul_rn(s, ay), sz = __dmul_rn(s, az);
    const double c1x = __dmul_rn(1.0 - c, ax), c1y = __dmul_rn(1.0 - c, ay), c1z = __dmul_rn(1.0 - c, az);
    double M[9];
    double tmp;
    tmp = __dmul_rn(c1x, ay); M[1] = tmp - sz; M[3] = tmp + sz;
    tmp = __dmul_rn(c1x, az); M[2] = tmp + sy; M[6] = tmp - sy;
    tmp = __dmul_rn(c1y, az); M[5] = tmp - sx; M[7] = tmp + sx;
    M[0] = __dadd_rn(__dmul_rn(c1x, ax), c); M[4] = __dadd_rn(__dmul_rn(c1y, ay), c); M[8] = __dadd_rn(__dmul_rn(c1z, az), c);
    float* o = Rt + 12 * f;
#pragma unroll
    for (int i = 0; i < 9; ++i) o[i] = static_cast<float>(M[i]);
    o[9] = static_cast<float>(poses[6 * f + 3]); o[10] = static_cast<float>(poses[6 * f + 4]); o[11] = static_cast<float>(poses[6 * f + 5]);
}

// per-frame pose constants (rotation matrix in both precisions, SO(3) right Jacobian, small-angle flag): computed once per
// state instead of once per row and sample point (the reference recomputes sin/cos in AngleAxisRotatePoint for each of the
// 4 points of every row and every Jet pass)
__global__ void k_frame_pose(int F, const double* __restrict__ poses, FramePose* __restrict__ out)
{
    pdl_prologue();
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    FramePose fp;
    frame_pose_make(poses + 6 * f, &fp);
    out[f] = fp;
}

struct SelectCam { float fx, fy, cx, cy; float d[5]; int dist_zero; float occlusion; };

// SDFColorization::computeObservation -> weight (float pipeline, exact rounding; see oracle.cpp observation_weight)
// pix (optional): Camera::project's sub-pixel position pt2f, for the colour lookup of the recolouring pass
__device__ __forceinline__ float observation_weight(const float pt[3], const float nrm[3], const float* __restrict__ Rt, const SelectCam& cam,
                                                    const float* __restrict__ depth, int W, int H, float* pix = nullptr)
{
    float q[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) q[k] = FA(FA(FA(FM(Rt[3 * k], pt[0]), FM(Rt[3 * k + 1], pt[1])), FM(Rt[3 * k + 2], pt[2])), Rt[9 + k]);
    float x = FD(q[0], q[2]);
    float y = FD(q[1], q[2]);
    if (!cam.dist_zero)
    {
        const float r2 = FA(FM(x, x), FM(y, y));
        const float r4 = FM(r2, r2);
        const float r6 = FM(r4, r2);
        const float dc = FA(FA(FA(1.0f, FM(cam.d[0], r2)), FM(cam.d[1], r4)), FM(cam.d[2], r6));
        const float xn = FA(FA(FM(x, dc), FM(FM(FM(2.0f, cam.d[3]), x), y)), FM(cam.d[4], FA(r2, FM(FM(2.0f, x), x))));
        const float yn = FA(FA(FM(y, dc), FM(FM(FM(2.0f, cam.d[4]), xn), y)), FM(cam.d[3], FA(r2, FM(FM(2.0f, y), y))));
        x = xn; y = yn;
    }
    const float pu = FA(FM(cam.fx, x), cam.cx);
    const float pv = FA(FM(cam.fy, y), cam.cy);
    if (pix) { pix[0] = pu; pix[1] = pv; }
    const float pu5 = FA(pu, 0.5f), pv5 = FA(pv, 0.5f);
    if (!(pu5 > -2147483000.0f && pu5 < 2147483000.0f && pv5 > -2147483000.0f && pv5 < 2147483000.0f)) return 0.0f;
    const int iu = __float2int_rz(pu5), iv = __float2int_rz(pv5);
    if (iu < 0 || iu >= W || iv < 0 || iv >= H) return 0.0f;
    const float d = __ldg(depth + static_cast<size_t>(iv) * W + iu);
    if (cam.occlusion > 0.0f)
    {
        if (!(d > 0.0f)) return 0.0f;
        const float sd = FS(d, q[2]);
        if (!(fabsf(sd) <= cam.occlusion)) return 0.0f;
    }
    if (d <= 0.0f) return 0.0f;
    float nc[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) nc[k] = FA(FA(FM(Rt[3 * k], nrm[0]), FM(Rt[3 * k + 1], nrm[1])), FM(Rt[3 * k + 2], nrm[2]));
    float w_normal = 0.0f;
    if (!(nc[0] == 0.0f && nc[1] == 0.0f && nc[2] == 0.0f))
    {
        const float qn2 = FA(FA(FM(q[0], q[0]), FM(q[1], q[1])), FM(q[2], q[2]));
        float v0 = q[0], v1 = q[1], v2 = q[2];
        if (qn2 > 0.0f) { const float ql = __fsqrt_rn(qn2); v0 = FD(q[0], ql); v1 = FD(q[1], ql); v2 = FD(q[2], ql); }
        const float dt = FA(FA(FM(v0, nc[0]), FM(v1, nc[1])), FM(v2, nc[2]));
        w_normal = FS(1.0f, fabsf(dt));
        w_normal = (1.0f < w_normal) ? 1.0f : w_normal;           // std::min(w_normal, 1.0f)
        w_normal = (w_normal < 0.0f) ? 0.0f : w_normal;           // std::max(.., 0.0f)
        const float div = FA(1.0f, FM(2.0f, w_normal));
        const float rk = FD(1.0f, FM(FM(div, div), div));
        w_normal = (rk < 0.001f) ? 0.001f : rk;
    }
    // depth weight: the reference computes max(1 - (clamp(d) - d_min)/(d_max - d_min), 1.0f), which is exactly 1.0f for
    // every finite d (Q1); w_normal * 1.0f == w_normal bit-for-bit, so the dead arithmetic is skipped.
    return w_normal;
}

// observation_weight() split at its one dependent load, for software pipelining in k_select_obs: obs_probe() transforms and projects
// the point and ISSUES the depth tap; obs_finish() consumes it.  Same operations in the same order as observation_weight()
// (the selection stays bit-identical; tests/test_gpu_parity.py, test_golden.py).
struct ObsProbe { float q0, q1, q2, d; int ok; };
__device__ __forceinline__ ObsProbe obs_probe(const float pt[3], const float* __restrict__ Rt, const SelectCam& cam, const float* __restrict__ depth, int W, int H)
{
    ObsProbe o;
    float q[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) q[k] = FA(FA(FA(FM(Rt[3 * k], pt[0]), FM(Rt[3 * k + 1], pt[1])), FM(Rt[3 * k + 2], pt[2])), Rt[9 + k]);
    o.q0 = q[0]; o.q1 = q[1]; o.q2 = q[2]; o.d = 0.0f; o.ok = 0;
    float x = FD(q[0], q[2]);
    float y = FD(q[1], q[2]);
    if (!cam.dist_zero)
    {
        const float r2 = FA(FM(x, x), FM(y, y));
        const float r4 = FM(r2, r2);
        const float r6 = FM(r4, r2);
        const float dc = FA(FA(FA(1.0f, FM(cam.d[0], r2)), FM(cam.d[1], r4)), FM(cam.d[2], r6));
        const float xn = FA(FA(FM(x, dc), FM(FM(FM(2.0f, cam.d[3]), x), y)), FM(cam.d[4], FA(r2, FM(FM(2.0f, x), x))));
        const float yn = FA(FA(FM(y, dc), FM(FM(FM(2.0f, cam.d[4]), xn), y)), FM(cam.d[3], FA(r2, FM(FM(2.0f, y), y))));
        x = xn; y = yn;
    }
    const float pu5 = FA(FA(FM(cam.fx, x), cam.cx), 0.5f), pv5 = FA(FA(FM(cam.fy, y), cam.cy), 0.5f);
    if (!(pu5 > -2147483000.0f && pu5 < 2147483000.0f && pv5 > -2147483000.0f && pv5 < 2147483000.0f)) return o;
    const int iu = __float2int_rz(pu5), iv = __float2int_rz(pv5);
    if (iu < 0 || iu >= W || iv < 0 || iv >= H) return o;
    o.d = __ldg(depth + static_cast<size_t>(iv) * W + iu);
    o.ok = 1;
    return o;
}
__device__ __forceinline__ float obs_finish(const ObsProbe& o, const float nrm[3], const float* __restrict__ Rt, const SelectCam& cam)
{
    if (!o.ok) return 0.0f;
    const float d = o.d;
    const float q[3] = {o.q0, o.q1, o.q2};
    if (cam.occlusion > 0.0f)
    {
        if (!(d > 0.0f)) return 0.0f;
        const float sd = FS(d, q[2]);
        if (!(fabsf(sd) <= cam.occlusion)) return 0.0f;
    }
    if (d <= 0.0f) return 0.0f;
    float nc[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) nc[k] = FA(FA(FM(Rt[3 * k], nrm[0]), FM(Rt[3 * k + 1], nrm[1])), FM(Rt[3 * k + 2], nrm[2]));
    float w_normal = 0.0f;
    if (!(nc[0] == 0.0f && nc[1] == 0.0f && nc[2] == 0.0f))
    {
        const float qn2 = FA(FA(FM(q[0], q[0]), FM(q[1], q[1])), FM(q[2], q[2]));
        float v0 = q[0], v1 = q[1], v2 = q[2];
        if (qn2 > 0.0f) { const float ql = __fsqrt_rn(qn2); v0 = FD(q[0], ql); v1 = FD(q[1], ql); v2 = FD(q[2], ql); }
        const float dt = FA(FA(FM(v0, nc[0]), FM(v1, nc[1])), FM(v2, nc[2]));
        w_normal = FS(1.0f, fabsf(dt));
        w_normal = (1.0f < w_normal) ? 1.0f : w_normal;
        w_normal = (w_normal < 0.0f) ? 0.0f : w_normal;
        const float div = FA(1.0f, FM(2.0f, w_normal));
        const float rk = FD(1.0f, FM(FM(div, div), div));
        w_normal = (rk < 0.001f) ? 0.001f : rk;
    }
    return w_normal;
}

// ---- conservative frame culling for the observation selection ---------------------------------------------------------
// Per frame, 32x32-pixel tiles of the depth map: minimum positive depth (+inf if none) and maximum depth.  Built once per
// i3d_upload_frames.  A warp of k_select_obs (32 consecutive active voxels = a compact spatial cluster when the grid is in a
// coherent order) bounds its iso-points by a sphere and asks, per frame: can ANY point of the sphere pass the reference's
// tests (pixel inside the image, d > 0, |d - z| <= occlusion)?  If not, every voxel of the warp has weight exactly 0 for
// that frame and the exact per-voxel computation is skipped.  The selection result is bit-identical by construction
// (only provably-zero weights are skipped); the parity tests check it.
constexpr int kCullTile = 32;
constexpr int kCullMaxWords = 16;     // frames / 32 handled by the culling mask (F <= 512); beyond that no culling

__global__ void k_depth_tiles(int F, int W, int H, const float* __restrict__ depth, float* __restrict__ tmin, float* __restrict__ tmax)
{
    const int TW = (W + kCullTile - 1) / kCullTile, TH = (H + kCullTile - 1) / kCullTile;
    const int t = blockIdx.x;                    // one block per tile
    if (t >= F * TW * TH) return;
    const int f = t / (TW * TH), r = t % (TW * TH), ty = r / TW, tx = r % TW;
    const float* img = depth + static_cast<size_t>(f) * W * H;
    float mn = __int_as_float(0x7f800000), mx = 0.0f;
    for (int i = threadIdx.x; i < kCullTile * kCullTile; i += blockDim.x)
    {
        const int px = tx * kCullTile + (i % kCullTile), py = ty * kCullTile + (i / kCullTile);
        if (px < W && py < H)
        {
            const float d = img[static_cast<size_t>(py) * W + px];
            if (d > 0.0f) { mn = fminf(mn, d); mx = fmaxf(mx, d); }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
    __shared__ float smn[8], smx[8];
    if ((threadIdx.x & 31) == 0) { smn[threadIdx.x >> 5] = mn; smx[threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x == 0)
    {
        for (int w = 1; w < (blockDim.x >> 5); ++w) { mn = fminf(mn, smn[w]); mx = fmaxf(mx, smx[w]); }
        tmin[t] = mn; tmax[t] = mx;
    }
}

struct CullView { const float* tmin; const float* tmax; int enabled; unsigned long long* stats; /* [0] frames visited, [1] frames total (per warp), optional */ };

// true = the frame may see some point of the sphere (centre c, radius rad), false = provably no voxel of the cluster is visible
__device__ __forceinline__ bool frame_may_see(const float c[3], float rad, const float* __restrict__ Rt, const SelectCam& cam, const CullView& cv,
                                              int f, int W, int H)
{
    const float qx = Rt[0] * c[0] + Rt[1] * c[1] + Rt[2] * c[2] + Rt[9];
    const float qy = Rt[3] * c[0] + Rt[4] * c[1] + Rt[5] * c[2] + Rt[10];
    const float qz = Rt[6] * c[0] + Rt[7] * c[1] + Rt[8] * c[2] + Rt[11];
    const float zmin = qz - rad, zmax = qz + rad;
    if (!(zmin > 1e-3f)) return true;                           // sphere touches the camera plane: no claim
    const float iz = 1.0f / qz;
    float xc = qx * iz, yc = qy * iz;
    // |x/z - xc/zc| <= rad (1 + |xc/zc|) / zmin per axis for every point of the sphere
    const float rnx = rad * (1.0f + fabsf(xc)) / zmin, rny = rad * (1.0f + fabsf(yc)) / zmin;
    float lip = 1.0f;
    if (!cam.dist_zero)
    {
        // lens distortion (Camera::project, y' uses the distorted x', Q2): map the centre exactly, bound the footprint growth by a
        // Lipschitz constant of the distortion map over the disk of normalised radius R that contains the footprint
        const float R = sqrtf(xc * xc + yc * yc) + 1.4143f * fmaxf(rnx, rny);
        const float R2 = R * R;
        const float grow = 3.0f * fabsf(cam.d[0]) * R2 + 5.0f * fabsf(cam.d[1]) * R2 * R2 + 7.0f * fabsf(cam.d[2]) * R2 * R2 * R2 +
                           8.0f * (fabsf(cam.d[3]) + fabsf(cam.d[4])) * R;
        lip = 1.0f + 2.0f * grow * (1.0f + 2.0f * fabsf(cam.d[4]) * R);      // generous: the y' term multiplies the x' growth once more
        const float r2 = xc * xc + yc * yc;
        const float dc = 1.0f + cam.d[0] * r2 + cam.d[1] * r2 * r2 + cam.d[2] * r2 * r2 * r2;
        const float xd = xc * dc + 2.0f * cam.d[3] * xc * yc + cam.d[4] * (r2 + 2.0f * xc * xc);
        const float yd = yc * dc + 2.0f * cam.d[4] * xd * yc + cam.d[3] * (r2 + 2.0f * yc * yc);
        xc = xd; yc = yd;
    }
    const float uc = cam.fx * xc + cam.cx, vc = cam.fy * yc + cam.cy;
    // + 2 px for the float pipeline's rounding and the nearest-pixel rounding
    const float ru = cam.fx * 1.4143f * fmaxf(rnx, rny) * lip * 1.001f + 2.0f;
    const float rv = cam.fy * 1.4143f * fmaxf(rnx, rny) * lip * 1.001f + 2.0f;
    if (uc + ru < 0.0f || uc - ru > static_cast<float>(W) || vc + rv < 0.0f || vc - rv > static_cast<float>(H)) return false;   // entirely outside
    const int TW = (W + kCullTile - 1) / kCullTile, TH = (H + kCullTile - 1) / kCullTile;
    const int tx0 = max(0, static_cast<int>(floorf((uc - ru) / kCullTile))), tx1 = min(TW - 1, static_cast<int>(floorf((uc + ru) / kCullTile)));
    const int ty0 = max(0, static_cast<int>(floorf((vc - rv) / kCullTile))), ty1 = min(TH - 1, static_cast<int>(floorf((vc + rv) / kCullTile)));
    if (tx1 - tx0 > 3 || ty1 - ty0 > 3) return true;            // large footprint: do not bother
    float dmin = __int_as_float(0x7f800000), dmax = 0.0f;
    const float* mn = cv.tmin + static_cast<size_t>(f) * TW * TH;
    const float* mx = cv.tmax + static_cast<size_t>(f) * TW * TH;
    for (int ty = ty0; ty <= ty1; ++ty)
        for (int tx = tx0; tx <= tx1; ++tx) { dmin = fminf(dmin, mn[ty * TW + tx]); dmax = fmaxf(dmax, mx[ty * TW + tx]); }
    if (!(dmax > 0.0f)) return false;                           // no positive depth under the footprint: computeWeight returns 0
    if (cam.occlusion > 0.0f)
    {
        const float tol = cam.occlusion * 1.001f + 1e-4f;
        if (zmin > dmax + tol || zmax < dmin - tol) return false;   // |d - z| <= occlusion impossible
    }
    return true;
}

// One thread per active voxel, serial loop over the candidate frames; the best K (weight, frame) keys are kept in a small
// sorted register list (key = weight bits << 32 | frame + 1: larger weight first, ties -> higher frame id = the
// canonical top-K of oracle.cpp).  Neighbouring threads are neighbouring voxels, so for a given frame the 32
// depth taps of a warp fall on neighbouring pixels, and the per-frame pose (R|t) is warp-uniform (shared memory
// broadcast).  Frames that provably see no voxel of the warp's cluster are skipped (frame_may_see).
#ifndef I3D_SELECT_PIPELINE
#define I3D_SELECT_PIPELINE 1
#endif
template <int KMAX>
__global__ void __launch_bounds__(kThreads)
k_select_obs(GridView g, FrameView fr, const float* __restrict__ Rt, SelectCam cam, CullView cull, int n_active, int stride,
             const int32_t* __restrict__ act, int K, int32_t* __restrict__ obs_frame /* [K][stride] */, float* __restrict__ obs_w /* [K][stride] */)
{
    pdl_prologue();
    extern __shared__ float s_rt[];     // [F][12]
    for (int i = threadIdx.x; i < 12 * fr.F; i += blockDim.x) s_rt[i] = Rt[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in_range = a < n_active;
    if (__ballot_sync(0xffffffffu, in_range) == 0u) return;     // whole warp past the end
    float nrm[3] = {0.0f, 0.0f, 0.0f};
    float pt[3] = {0.0f, 0.0f, 0.0f};
    if (in_range)
    {
        const int64_t v = act[a];
        surface_normal_f(g, v, nrm);
        const float s = static_cast<float>(g.sdf[v]);
        pt[0] = FS(FM(static_cast<float>(g.x[v]), g.voxel_size), FM(nrm[0], s));
        pt[1] = FS(FM(static_cast<float>(g.y[v]), g.voxel_size), FM(nrm[1], s));
        pt[2] = FS(FM(static_cast<float>(g.z[v]), g.voxel_size), FM(nrm[2], s));
    }
    // ---- bounding sphere of the warp's iso-points, then the candidate-frame mask (lane l tests frames l, l+32, ...)
    const int nwords = (fr.F + 31) / 32;
    __shared__ unsigned s_mask[kThreads / 32][kCullMaxWords];   // candidate-frame bit mask per warp (one copy of the visiting loop: no unrolling)
    unsigned* wmask = s_mask[threadIdx.x >> 5];
    const bool culling = cull.enabled && nwords <= kCullMaxWords;
    if (culling)
    {
        const float big = 3.0e38f;
        float lo[3], hi[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) { lo[k] = in_range ? pt[k] : big; hi[k] = in_range ? pt[k] : -big; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int k = 0; k < 3; ++k) { lo[k] = fminf(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o)); hi[k] = fmaxf(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o)); }
        const float c[3] = {0.5f * (lo[0] + hi[0]), 0.5f * (lo[1] + hi[1]), 0.5f * (lo[2] + hi[2])};
        const float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        const float rad = 0.5f * sqrtf(dx * dx + dy * dy + dz * dz) * 1.001f + 1e-4f;
#pragma unroll 1
        for (int j = 0; j < nwords; ++j)
        {
            const int f = 32 * j + lane;
            const bool may = (f < fr.F) && frame_may_see(c, rad, s_rt + 12 * f, cam, cull, f, fr.W, fr.H);
            const unsigned m = __ballot_sync(0xffffffffu, may);
            if (lane == 0) wmask[j] = m;
        }
        __syncwarp();
    }
    const size_t img = static_cast<size_t>(fr.W) * fr.H;
    unsigned long long best[KMAX];
#pragma unroll
    for (int k = 0; k < KMAX; ++k) best[k] = 0ull;
    auto insert = [&](float wf, int f) {
        if (wf > 0.0f && in_range)
        {
            unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(wf)) << 32) | static_cast<unsigned>(f + 1);
            // sorted insertion (descending); slots >= K are never read
#pragma unroll
            for (int k = 0; k < KMAX; ++k)
            {
                const unsigned long long hi2 = key > best[k] ? key : best[k];
                const unsigned long long lo2 = key > best[k] ? best[k] : key;
                best[k] = hi2; key = lo2;
            }
        }
    };
    if (cull.stats && lane == 0)
    {
        unsigned long long vis = 0;
        for (int j = 0; j < nwords; ++j) vis += culling ? __popc(wmask[j]) : 32;
        atomicAdd(cull.stats, vis); atomicAdd(cull.stats + 1, static_cast<unsigned long long>(fr.F));
    }
    // The visiting loop is a serial chain of (transform, project, DEPENDENT depth tap, weight, insert) per candidate frame; with a shard
    // of the grid per GPU the whole launch is a single wave and its duration is the longest such chain (0.29 ms for 1/8 of the C3 grid
    // against 1.0 ms for all of it, profiles/r02s_bench_c3_8gpu_p2p.json).  Software pipelining, depth 2: the depth tap of frame i+1
    // is issued (obs_probe) before the weight of frame i is finished (obs_finish), so the tap's latency overlaps a visit's arithmetic.
    ObsProbe pend; pend.ok = 0; pend.q0 = pend.q1 = pend.q2 = pend.d = 0.0f;
    int pend_f = -1;
#pragma unroll 1
    for (int j = 0; j < nwords; ++j)
    {
        unsigned m = culling ? wmask[j] : 0xffffffffu;          // warp-uniform
#pragma unroll 1
        while (m)
        {
            const int f = 32 * j + __ffs(m) - 1;
            m &= m - 1;
            if (f >= fr.F) continue;
#if I3D_SELECT_PIPELINE
            const ObsProbe nxt = obs_probe(pt, s_rt + 12 * f, cam, fr.depth + img * f, fr.W, fr.H);
            if (pend_f >= 0) insert(obs_finish(pend, nrm, s_rt + 12 * pend_f, cam), pend_f);
            pend = nxt; pend_f = f;
#else
            insert(observation_weight(pt, nrm, s_rt + 12 * f, cam, fr.depth + img * f, fr.W, fr.H), f);
#endif
        }
    }
    if (pend_f >= 0) insert(obs_finish(pend, nrm, s_rt + 12 * pend_f, cam), pend_f);
    if (!in_range) return;
    // Slot order carries no meaning for the solve; order the K selected observations by ascending frame id so that
    // neighbouring voxels (which mostly select the same frames, in varying rank order) agree slot by slot: the
    // per-frame warp reductions of k_eg_accum / k_eg_apply then see ~1 distinct frame per warp and slot.
    // Re-key as (frame+1) << 32 | weight bits; empty entries (0) sort last.
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
    {
        if (k >= K || best[k] == 0ull) best[k] = ~0ull;
        else best[k] = ((best[k] & 0xffffffffull) << 32) | (best[k] >> 32);
    }
#pragma unroll
    for (int i = 0; i < KMAX; ++i)
#pragma unroll
        for (int j = 0; j + 1 < KMAX - i; ++j)
        {
            const unsigned long long lo = best[j] < best[j + 1] ? best[j] : best[j + 1];
            const unsigned long long hi = best[j] < best[j + 1] ? best[j + 1] : best[j];
            best[j] = lo; best[j + 1] = hi;
        }
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
    {
        if (k >= K) break;
        int fsel = -1; float wsel = 0.0f;
        if (best[k] != ~0ull) { fsel = static_cast<int>(best[k] >> 32) - 1; wsel = __uint_as_float(static_cast<unsigned>(best[k] & 0xffffffffull)); }
        obs_frame[static_cast<size_t>(k) * stride + a] = fsel;
        obs_w[static_cast<size_t>(k) * stride + a] = wsel;
    }
}

// ----------------------------------------------------------------------------------------------
// k2: E_g residual + Jacobian build (ShadingCost::create + functor; shading_cost.cpp:59-150, shading_cost.h:85-198)
// ----------------------------------------------------------------------------------------------
struct CamView
{
    const double* cam;               // poses[6F] | intr[4] | dist[5]
    const FramePose* fpose;          // [F], from k_frame_pose for the same poses
    int F;
};

struct EgRows
{
    int n_active, K;
    int stride;            // slots per k (n_active rounded up to 64): slot = k*stride + a; keeps every column segment 256 B aligned for bulk copies
    const int32_t* act;
    float* J;              // [29][K*n_a]
    int32_t* row_frame;    // [K*n_a] valid rows: frame, else -1
    double* row_res;       // unweighted residual
    double* row_wraw;      // raw weight = obs.weight * sdfToWeight
    float* row_w;          // final weight (raw * type weight)
};

__device__ __forceinline__ void make_cam_params(const CamView& cv, double pyr_scale, int W, int H, CamParams<double>* c)
{
    const double* intr = cv.cam + 6 * cv.F;
    const double* dist = intr + 4;
    c->fx = intr[0] * pyr_scale; c->fy = intr[1] * pyr_scale; c->cx = intr[2] * pyr_scale; c->cy = intr[3] * pyr_scale;
    c->k1 = dist[0]; c->k2 = dist[1]; c->k3 = dist[2]; c->p1 = dist[3]; c->p2 = dist[4];
    c->pyr_scale = pyr_scale; c->w = W; c->h = H;
}

// gathers the 10 sdf + 4 albedo parameters of voxel v's E_g stencil; returns false if a stencil voxel is absent
__device__ __forceinline__ bool gather_stencil(const GridView& g, const double* __restrict__ sdf, const double* __restrict__ alb, int64_t v,
                                               int32_t idx[14], double s10[10], double a4[4])
{
    const int64_t n = g.n;
    const int32_t xp = g.nbr[NB_XP * n + v], yp = g.nbr[NB_YP * n + v], zp = g.nbr[NB_ZP * n + v];
    const int32_t x2 = g.nbr[NB_X2 * n + v], y2 = g.nbr[NB_Y2 * n + v], z2 = g.nbr[NB_Z2 * n + v];
    const int32_t xy = g.nbr[NB_XY * n + v], xz = g.nbr[NB_XZ * n + v], yz = g.nbr[NB_YZ * n + v];
    // parameter order of the reference: (0,0,0) (0,1,0) (0,2,0) (0,1,1) (0,0,1) (0,0,2) (1,0,0) (1,1,0) (1,0,1) (2,0,0)
    idx[0] = static_cast<int32_t>(v); idx[1] = yp; idx[2] = y2; idx[3] = yz; idx[4] = zp; idx[5] = z2; idx[6] = xp; idx[7] = xy; idx[8] = xz; idx[9] = x2;
    idx[10] = static_cast<int32_t>(v); idx[11] = xp; idx[12] = yp; idx[13] = zp;
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 10; ++k) ok = ok && (idx[k] >= 0);
    if (!ok) return false;
#pragma unroll
    for (int k = 0; k < 10; ++k) s10[k] = sdf[idx[k]];
#pragma unroll
    for (int k = 0; k < 4; ++k) a4[k] = alb[idx[10 + k]];
    return true;
}

// SDFOperators::sdfToWeight (src/sdf/operators.cpp:142-147)
__device__ __forceinline__ double sdf_to_weight(double sdf, double truncation)
{
    const double a = fmin(fabs(sdf), truncation) / truncation;
    return fmin(fmax(1.0 - a, 0.01), 1.0);
}

// camera-block accumulators in shared memory: per frame 6 (gradient) + 6 (column norms) + 21 (6x6 upper) ;
// then 9 + 9 + 10 + 15 for intrinsics/distortion.  Layout helper.
struct CamAccLayout
{
    int F;
    __host__ __device__ int pose_stride() const { return 33; }
    __host__ __device__ int tail() const { return 33 * F; }          // intr/dist part: 9 grad + 9 colsq + 10 + 15
    __host__ __device__ int size() const { return 33 * F + 43; }
};

// k2a / k7: the E_g rows of one voxel, owned by ONE thread (round 2; round 1 ran one thread per row slot, k-major, and
// re-gathered the 14-entry stencil, 72 B of SH and the neighbour ids in five different warps: DRAM reads 5x algorithmic,
// profiles/r01c_final_k_eg_build.csv).  Per voxel, once: stencil gather, the four normals / shading values / iso-points
// (voxel_geom_make, float64).  Per selected frame: rigid transform, projection with distortion, bicubic luminance
// (float64 value, float32 gradient), then
//   ROWS_BUILD: the 29-column row by the closed-form chain rule (float32) -> raw J row (column-major: every store of a
//               warp is one full 128 B line), unweighted residual, raw weight
//   ROWS_COST : sum of raw_weight * r^2 at an arbitrary state (rows fixed at creation; invalid -> 0 like the functor)
// Neighbouring threads are neighbouring voxels of the compacted active list: their stencil gathers hit the same lines, they
// mostly select the same frame in the same slot (k_select_obs orders slots by frame id), so the per-frame constants are
// warp-broadcast loads and the 16 luminance taps of a warp fall on neighbouring pixels.
enum { ROWS_BUILD = 0, ROWS_COST = 1 };
constexpr int kRowThreads = 128;       // block size of the global-memory variant of k_eg_rows (256 for the staged variant)
#ifndef I3D_ROWS_STAGE_POSE
#define I3D_ROWS_STAGE_POSE 1          // 0: never stage the pose table (A/B switch)
#endif

// ---- bulk-async copy (cp.async.bulk, the non-tensor TMA path) + mbarrier, used to stage the per-frame pose table ----------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes /* multiple of 16 */, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t done = 0;
    while (!done)
        asm volatile("{\n\t.reg .pred P1;\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\tselp.b32 %0, 1, 0, P1;\n\t}"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
}

// dynamic shared memory of k_eg_rows: [mbarrier | pose table F x 176 B (STAGE only)] [VoxelGeom columns] [VoxelDeriv columns (BUILD only)]
__host__ __device__ inline size_t rows_pose_bytes(int F) { return (static_cast<size_t>(F) * sizeof(FramePose) + 127) & ~static_cast<size_t>(127); }
__host__ __device__ inline size_t rows_smem_bytes(int mode, int threads, bool stage, int F)
{
    return (stage ? 128 + rows_pose_bytes(F) : 0) + static_cast<size_t>(threads) * (kVoxelGeomWords * sizeof(double) + (mode == ROWS_BUILD ? kVoxelDerivWords * sizeof(float) : 0));
}

// THREADS / STAGE: 128 threads x 4 blocks per SM reading the pose constants from global memory (L1), or — when the table of all F
// frames fits next to two 256-thread blocks' state (F <= ~230) — 256 threads x 2 blocks per SM with the whole table staged into
// shared memory by ONE bulk-async copy per block (cp.async.bulk + mbarrier: issued by thread 0 right after the grid dependency
// resolves, complete long before the stencil gather and the voxel geometry are done), so that a row's pose constants are LDS reads
// that depend on nothing but the frame id.  Same occupancy (16 warps per SM, 128 registers) in both variants.
template <int MODE, int THREADS, bool STAGE>
__global__ void __launch_bounds__(THREADS, THREADS == 128 ? 4 : 2)
k_eg_rows(GridView g, FrameView fr, CamView cv, EgRows rows, const int32_t* __restrict__ obs_frame, const float* __restrict__ obs_w, ReduceSite site)
{
    extern __shared__ __align__(128) unsigned char s_rows[];
    pdl_prologue();
    uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_rows);
    const FramePose* s_pose = reinterpret_cast<const FramePose*>(s_rows + 128);
    unsigned char* s_state = s_rows + (STAGE ? 128 + rows_pose_bytes(fr.F) : 0);
    double* s_vg = reinterpret_cast<double*>(s_state);                                            // [kVoxelGeomWords][THREADS]
    float* s_vd = reinterpret_cast<float*>(s_state + static_cast<size_t>(THREADS) * kVoxelGeomWords * sizeof(double));   // [kVoxelDerivWords][THREADS]
    if (STAGE)
    {
        if (threadIdx.x == 0)
        {
            const uint32_t bytes = static_cast<uint32_t>(fr.F * sizeof(FramePose));
            mbar_init(s_bar, 1);
            mbar_expect_tx(s_bar, bytes);
            bulk_copy_g2s(s_rows + 128, cv.fpose, bytes, s_bar);
        }
        __syncthreads();          // the barrier object is initialised before anyone polls it
    }
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    const size_t S = static_cast<size_t>(rows.K) * rows.stride;
    double acc[1] = {0.0};
    // per-voxel state of the frame loop parked in shared memory (15 doubles + 40 floats per thread)
    const VoxelGeomView vg{s_vg + threadIdx.x, THREADS};
    const VoxelDerivView vd{s_vd + threadIdx.x, THREADS};
    bool ok = a < rows.n_active;
    double wsdf = 0.0;
    if (ok)
    {
        const int64_t v = rows.act[a];
        int32_t idx[14];
        double s10[10], a4[4];
        ok = gather_stencil(g, g.sdf, g.albedo, v, idx, s10, a4);
        if (ok)
        {
            double sh[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) sh[k] = g.sh[static_cast<int64_t>(k) * g.n + v];
            const int coord[3] = {g.x[v], g.y[v], g.z[v]};
            VoxelGeom vg_r;
            VoxelDeriv vd_r;
            voxel_geom_make<MODE == ROWS_BUILD>(s10, a4, coord, static_cast<double>(g.voxel_size), sh, &vg_r, &vd_r);
            voxel_geom_park(vg_r, s_vg + threadIdx.x, THREADS);
            if (MODE == ROWS_BUILD) voxel_deriv_park(vd_r, s_vd + threadIdx.x, THREADS);
            if (MODE == ROWS_BUILD) wsdf = sdf_to_weight(s10[0], static_cast<double>(g.truncation));
        }
    }
    if (STAGE) mbar_wait(s_bar, 0);
    if (a < rows.stride)
    {
        CamParams<double> cam;
        make_cam_params(cv, fr.pyr_scale, fr.W, fr.H, &cam);
        const size_t img_stride = static_cast<size_t>(fr.W) * fr.H;
        const int32_t* __restrict__ fsrc = (MODE == ROWS_BUILD) ? obs_frame : rows.row_frame;
        int f_next = ok ? fsrc[a] : -1;
#pragma unroll 1
        for (int k = 0; k < rows.K; ++k)
        {
            const size_t slot = static_cast<size_t>(k) * rows.stride + a;
            const int f = f_next;
            if (ok && k + 1 < rows.K) f_next = fsrc[slot + rows.stride];      // prefetch: the frame id gates everything of the next row
            // ... and (global-memory variant) its pose constants (176 B, two lines) are requested into L1 one iteration ahead
            if (!STAGE && f_next >= 0)
            {
                const char* pf = reinterpret_cast<const char*>(cv.fpose + f_next);
                asm volatile("prefetch.global.L1 [%0];" ::"l"(pf));
                asm volatile("prefetch.global.L1 [%0];" ::"l"(pf + 128));
            }
            int32_t rf = -1; double res = 0.0, wraw = 0.0;
            if (f >= 0)
            {
                const FramePose& fp = STAGE ? s_pose[f] : cv.fpose[f];
                PointSave sv[4];
                float e[4];
                res = eg_frame_primal<MODE == ROWS_BUILD>(vg, fp, cam, LinearImage{fr.lum + img_stride * f}, sv, e);
                if (MODE == ROWS_BUILD)
                {
                    if (res != 0.0)
                    {
                        CamParams<float> cf;
                        cf.fx = static_cast<float>(cam.fx); cf.fy = static_cast<float>(cam.fy); cf.cx = static_cast<float>(cam.cx); cf.cy = static_cast<float>(cam.cy);
                        cf.k1 = static_cast<float>(cam.k1); cf.k2 = static_cast<float>(cam.k2); cf.k3 = static_cast<float>(cam.k3);
                        cf.p1 = static_cast<float>(cam.p1); cf.p2 = static_cast<float>(cam.p2);
                        cf.pyr_scale = static_cast<float>(cam.pyr_scale); cf.w = cam.w; cf.h = cam.h;
                        float row[29];
                        eg_frame_deriv(vd, fp, cf, sv, e, row);
                        rf = f;
                        wraw = static_cast<double>(obs_w[slot]) * wsdf;
                        float* __restrict__ jc = rows.J + slot;
#pragma unroll
                        for (int m = 0; m < 29; ++m) jc[static_cast<size_t>(m) * S] = row[m];
                    }
                }
                else acc[0] += rows.row_wraw[slot] * res * res;
            }
            if (MODE == ROWS_BUILD) { rows.row_frame[slot] = rf; rows.row_res[slot] = res; rows.row_wraw[slot] = wraw; }
        }
    }
    if (MODE == ROWS_COST) grid_reduce<1>(acc, site);
}

// k2b: accumulations over the freshly built rows (one thread per active voxel, J read back coalesced):
//   bg[j]  += w_raw * r * J[j]      (gradient, unscaled)         cg[j] += w_raw * J[j]^2   (column norms)
//   camera blocks (pose 6x6 per frame, intrinsics 4x4, distortion 5x5) += w_raw * J_a J_b
// The per-type weight (lambda/sum*1000) multiplies all of these later (it needs the global weight sum).
// Per-frame sums never go through contended shared-memory atomics (a float atomicAdd on shared memory is a CAS loop and
// neighbouring voxels mostly select the same frame): intrinsics/distortion products are summed per thread over the K rows
// and reduce-scattered once per warp; for the pose blocks each thread parks (6 pose entries, w, w*r) per row in shared
// memory, then the warp walks over the DISTINCT frames among its 32 x K rows and reduces the 33 products of each with a
// 32-wide butterfly reduce-scatter + one scalar all-reduce.
__global__ void __launch_bounds__(kThreads)
k_eg_accum(GridView g, EgRows rows, int F, double* __restrict__ bg, double* __restrict__ cg, double* __restrict__ cam_acc /* CamAccLayout.size() */,
           ReduceSite site /* out: [0] sum raw weights, [1] sum raw w*r^2, [2] valid rows */)
{
    // summed in double like k_eg_apply (same exactness condition on the block partials of the camera sums); k_acc_to_float
    // rounds the totals once
    pdl_prologue();
    extern __shared__ double s_dyn_d[];
    const CamAccLayout lay{F};
    double* s_cam = s_dyn_d;
    float* s_park = reinterpret_cast<float*>(s_dyn_d + ((lay.size() + 15) & ~15));   // [K][8][kThreads]
    for (int i = threadIdx.x; i < lay.size(); i += blockDim.x) s_cam[i] = 0.0;
    __syncthreads();
    const int tid = threadIdx.x, lane = tid & 31;
    const int a = blockIdx.x * blockDim.x + tid;
    const bool in_range = a < rows.n_active;
    const size_t S = static_cast<size_t>(rows.K) * rows.stride;
    double acc[3] = {0.0, 0.0, 0.0};
    float gsum[14], csum[14];
#pragma unroll
    for (int m = 0; m < 14; ++m) { gsum[m] = 0.0f; csum[m] = 0.0f; }
    float tl[64];                                             // 9 grad, 9 colsq, 10 + 15 upper triangles of the intrinsics / distortion blocks
#pragma unroll
    for (int i = 0; i < 64; ++i) tl[i] = 0.0f;
    int fk[I3D_MAX_OBS];
#pragma unroll
    for (int k = 0; k < I3D_MAX_OBS; ++k)
    {
        fk[k] = -1;
        if (k >= rows.K) continue;
        const size_t slot = static_cast<size_t>(k) * rows.stride + (in_range ? a : 0);
        const int f = in_range ? rows.row_frame[slot] : -1;
        fk[k] = f;
        if (f >= 0)
        {
            float row[29];
#pragma unroll
            for (int m = 0; m < 29; ++m) row[m] = rows.J[static_cast<size_t>(m) * S + slot];
            const double wraw = rows.row_wraw[slot], res = rows.row_res[slot];
            const float wf = static_cast<float>(wraw), wr = static_cast<float>(wraw * res);
            acc[0] += wraw; acc[1] += wraw * res * res; acc[2] += 1.0;
#pragma unroll
            for (int m = 0; m < 14; ++m) { gsum[m] += wr * row[m]; csum[m] += wf * row[m] * row[m]; }
#pragma unroll
            for (int m = 0; m < 9; ++m) { tl[m] += wr * row[20 + m]; tl[9 + m] += wf * row[20 + m] * row[20 + m]; }
            int t = 18;
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = r; c < 4; ++c) tl[t++] += wf * row[20 + r] * row[20 + c];
#pragma unroll
            for (int r = 0; r < 5; ++r)
#pragma unroll
                for (int c = r; c < 5; ++c) tl[t++] += wf * row[24 + r] * row[24 + c];
#pragma unroll
            for (int c = 0; c < 6; ++c) s_park[(k * 8 + c) * kThreads + tid] = row[14 + c];
            s_park[(k * 8 + 6) * kThreads + tid] = wf;
            s_park[(k * 8 + 7) * kThreads + tid] = wr;
        }
    }
    // ---- intrinsics / distortion: one reduce-scatter per warp
    if (__ballot_sync(0xffffffffu, acc[2] > 0.0) != 0u)
    {
        warp_reduce_scatter<64>(tl, lane);
#pragma unroll
        for (int i = 0; i < 2; ++i)
        {
            const int id = rs_index<64>(i, lane);
            if (id < 43 && tl[i] != 0.0f) atomicAdd(s_cam + lay.tail() + id, static_cast<double>(tl[i]));
        }
    }
    // ---- pose blocks: walk over the distinct frames of the warp's rows
    unsigned todo = 0u;
#pragma unroll
    for (int k = 0; k < I3D_MAX_OBS; ++k) if (fk[k] >= 0) todo |= 1u << k;
    while (true)
    {
        const unsigned pending = __ballot_sync(0xffffffffu, todo != 0u);
        if (pending == 0u) break;
        const int leader = __ffs(pending) - 1;
        const int mine_f = (todo != 0u) ? fk_select(fk, __ffs(todo) - 1) : -1;
        const int f0 = __shfl_sync(0xffffffffu, mine_f, leader);
        float jp[6] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
        float wf = 0.0f, wr = 0.0f;
#pragma unroll
        for (int k = 0; k < I3D_MAX_OBS; ++k)
        {
            if (k >= rows.K) break;
            if (((todo >> k) & 1u) && fk[k] == f0)
            {
#pragma unroll
                for (int c = 0; c < 6; ++c) jp[c] = s_park[(k * 8 + c) * kThreads + tid];
                wf = s_park[(k * 8 + 6) * kThreads + tid];
                wr = s_park[(k * 8 + 7) * kThreads + tid];
                todo &= ~(1u << k);
            }
        }
        // 33 products: 6 gradient, 6 column norms, 21 upper triangle; the first 32 via reduce-scatter, the last via all-reduce
        float v[32];
#pragma unroll
        for (int c = 0; c < 6; ++c) { v[c] = wr * jp[c]; v[6 + c] = wf * jp[c] * jp[c]; }
        int t = 12;
        float last = 0.0f;
#pragma unroll
        for (int r = 0; r < 6; ++r)
#pragma unroll
            for (int c = r; c < 6; ++c)
            {
                const float pr = wf * jp[r] * jp[c];
                if (t < 32) v[t] = pr; else last = pr;
                ++t;
            }
        warp_reduce_scatter<32>(v, lane);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) last += __shfl_xor_sync(0xffffffffu, last, o);
        double* dst = s_cam + lay.pose_stride() * f0;
        if (v[0] != 0.0f) atomicAdd(dst + lane, static_cast<double>(v[0]));              // rs_index<32>(0, lane) == lane
        if (lane == 0 && last != 0.0f) atomicAdd(dst + 32, static_cast<double>(last));
    }
    if (in_range && acc[2] > 0.0)
    {
        const int64_t v = rows.act[a];
        const int64_t n = g.n;
        const int32_t xp = g.nbr[NB_XP * n + v], yp = g.nbr[NB_YP * n + v], zp = g.nbr[NB_ZP * n + v];
        int64_t idx[14];
        idx[0] = v; idx[1] = yp; idx[2] = g.nbr[NB_Y2 * n + v]; idx[3] = g.nbr[NB_YZ * n + v]; idx[4] = zp; idx[5] = g.nbr[NB_Z2 * n + v];
        idx[6] = xp; idx[7] = g.nbr[NB_XY * n + v]; idx[8] = g.nbr[NB_XZ * n + v]; idx[9] = g.nbr[NB_X2 * n + v];
        idx[10] = n + v; idx[11] = n + xp; idx[12] = n + yp; idx[13] = n + zp;
#pragma unroll
        for (int m = 0; m < 14; ++m)
            if (csum[m] != 0.0f) { atomicAdd(bg + idx[m], static_cast<double>(gsum[m])); atomicAdd(cg + idx[m], static_cast<double>(csum[m])); }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < lay.size(); i += blockDim.x) { const float vv = static_cast<float>(s_cam[i]); if (vv != 0.0f) atomicAdd(cam_acc + i, static_cast<double>(vv)); }
    grid_reduce<3>(acc, site);
}

// k_eg_accum's double totals -> the float vectors the iteration reads
__global__ void k_acc_to_float(int64_t U, int ncam, const double* __restrict__ bgd, const double* __restrict__ cgd, const double* __restrict__ camd,
                               float* __restrict__ bg, float* __restrict__ cg, float* __restrict__ cam_acc)
{
    pdl_prologue();
    const int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (j < U) { bg[j] = static_cast<float>(bgd[j]); cg[j] = static_cast<float>(cgd[j]); }
    if (j < ncam) cam_acc[j] = static_cast<float>(camd[j]);
}

// final per-row weights once the type weight is known (NLSSolver::normalizeCostTermWeights, nls_solver.cpp:379-394)
__global__ void k_row_weights(size_t S, const double* __restrict__ row_wraw, const double* __restrict__ type_w, float* __restrict__ row_w)
{
    pdl_prologue();
    const size_t s = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    if (s >= S) return;
    row_w[s] = static_cast<float>(row_wraw[s] * type_w[0]);
}

// ----------------------------------------------------------------------------------------------
// regulariser rows (E_r, E_s, E_a): values, weight sums, costs
// ----------------------------------------------------------------------------------------------
struct RegView
{
    const uint8_t* flags;
    float* ea_w;             // [3][n] raw pair weight of {v, v+e_d}, 0 = no pair
    double* lap;             // [n] E_r residual (0 where no row)
    int use_er, use_es, use_ea;
};

__device__ __forceinline__ float intensity_u8(uchar4 c) { return FA(FA(FM(0.299f, static_cast<float>(c.x)), FM(0.587f, static_cast<float>(c.y))), FM(0.114f, static_cast<float>(c.z))); }

// AlbedoRegularizer::create weight (albedo_regularizer.cpp:60-72): returns false for NaN/Inf (pair skipped)
__device__ __forceinline__ bool albedo_pair_weight(uchar4 ca, uchar4 cb, float* w)
{
    const float la = intensity_u8(ca), lb = intensity_u8(cb);
    const float k = 1.0f / 255.0f;
    const float d0 = FS(FD(FM(static_cast<float>(ca.x), k), la), FD(FM(static_cast<float>(cb.x), k), lb));
    const float d1 = FS(FD(FM(static_cast<float>(ca.y), k), la), FD(FM(static_cast<float>(cb.y), k), lb));
    const float d2 = FS(FD(FM(static_cast<float>(ca.z), k), la), FD(FM(static_cast<float>(cb.z), k), lb));
    float chroma = __fsqrt_rn(FA(FA(FM(d0, d0), FM(d1, d1)), FM(d2, d2)));
    const float t = FS(1.0f, chroma);
    chroma = (t < 0.01f) ? 0.01f : t;        // std::max(t, 0.01f): NaN stays NaN
    if (isnan(chroma) || isinf(chroma)) return false;
    *w = chroma;
    return true;
}

// E_r / E_s / E_a rows at the current state: lap[], ea_w[], and per-type (count, weight sum, raw cost) partials.
// out: [0] n_Er  [1] sum r_Er^2  [2] n_Es  [3] sum r_Es^2  [4] n_Ea  [5] sum w_Ea  [6] sum w_Ea r^2  [7] n_free_sdf [8] n_free_alb
__global__ void __launch_bounds__(kThreads)
k_reg_build(GridView g, RegView rv, Shard sh, ReduceSite site)
{
    pdl_prologue();
    const int64_t vbase = sh.loc_begin + (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) * 4;
    double acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int e4 = 0; e4 < 4; ++e4)
    {
        const int64_t v = vbase + e4;
        if (v >= sh.loc_end) break;
        const uint8_t fl = rv.flags[v];
        const bool active = fl & FL_ACTIVE, ring = fl & FL_RING;
        const bool own = sh.owns_voxel(v);      // lap / ea_w are produced for every voxel, the sums only for owned rows
        if (own && (fl & FL_FREE_SDF)) acc[7] += 1.0;
        if (own && (fl & FL_FREE_ALB)) acc[8] += 1.0;
        double lap = 0.0;
        if (rv.use_er && active && ring)
        {
            const double c = g.sdf[v];
            const double xp = g.sdf[g.nbr[NB_XP * g.n + v]], xm = g.sdf[g.nbr[NB_XM * g.n + v]];
            const double yp = g.sdf[g.nbr[NB_YP * g.n + v]], ym = g.sdf[g.nbr[NB_YM * g.n + v]];
            const double zp = g.sdf[g.nbr[NB_ZP * g.n + v]], zm = g.sdf[g.nbr[NB_ZM * g.n + v]];
            lap = ((xp + xm - 2.0 * c) + (yp + ym - 2.0 * c)) + (zp + zm - 2.0 * c);
            if (own) { acc[0] += 1.0; acc[1] += lap * lap; }
        }
        rv.lap[v] = lap;
        if (rv.use_es && active && own)
        {
            double r = g.sdf[v] - g.sdf0[v];
            if (r == 0.0) r = 0.0000001;
            acc[2] += 1.0; acc[3] += r * r;
        }
        // pairs {v, v+e_d}, d = x,y,z.  Owner = the voxel whose addVoxelResiduals call creates the row (optimizer.cpp:259-276)
#pragma unroll
        for (int d = 0; d < 3; ++d)
        {
            float w = 0.0f;
            const int32_t b = g.nbr[static_cast<int64_t>(2 * d) * g.n + v];
            if (rv.use_ea && b >= 0)
            {
                const uint8_t fb = rv.flags[b];
                const bool act_b = fb & FL_ACTIVE, ring_b = fb & FL_RING;
                // v < b always in index terms? not necessarily: compare indices
                bool exists;
                if (active && act_b) exists = (v < b) ? ring : ring_b;       // the earlier one decides (Q6)
                else if (active) exists = ring;
                else if (act_b) exists = ring_b;
                else exists = false;
                if (exists && (fl & FL_VALID) && (fb & FL_VALID))
                {
                    float pw;
                    if (albedo_pair_weight(g.rgb[v], g.rgb[b], &pw) && pw != 0.0f)
                    {
                        w = pw;
                        const double r = g.albedo[v] - g.albedo[b];
                        if (own) { acc[4] += 1.0; acc[5] += static_cast<double>(pw); acc[6] += static_cast<double>(pw) * r * r; }
                    }
                }
            }
            rv.ea_w[static_cast<int64_t>(d) * g.n + v] = w;
        }
    }
    grid_reduce<9>(acc, site);
}

// ----------------------------------------------------------------------------------------------
// solver vectors
// ----------------------------------------------------------------------------------------------
struct SolveVecs
{
    int64_t n; int F; int64_t U;
    // problem constants (per GN iteration)
    float* bg;      // E_g gradient accumulation (unscaled, raw weights)
    float* cg;      // E_g column norms (raw weights)
    float* s;       // Jacobi column scale (0 for fixed unknowns)
    float* jtj;     // s^2 * colnorm^2  (diag of scaled J^T J)
    float* b;       // J'^T f
    // PCG
    float* x; float* r; float* z; float* p; float* ps; float* qg;
    double* qgd;    // [U] E_g part of qg in double (k_eg_apply), consumed and cleared by k_op_partial
    float* tr;      // [n] E_r row values of the current input vector (unweighted)
};

struct TypeWeights { double w[4]; };     // final per-type weights lambda/sum*1000

struct CgCtl
{
    // device-resident PCG state (ConjugateGradientsSolver::Solve restated, see oracle.cpp)
    double rho, last_rho, beta, alpha, pq, Q0, Q1, zeta;
    double xd2x;         // x . D^2 x of the current iterate (for the model cost change)
    double inv_radius;
    int it;              // completed iterations
    int done;            // 1 = stop (kernels become no-ops)
    int halt;            // sticky: the LM loop is over (set by k_lm_begin); the PCG init epilogue must not clear `done`
    int status;          // 0 running/success 1 failure(rho/beta/alpha) 2 indefinite (pq<=0) 3 max iterations
    int forced_iterations, max_iterations, min_iterations;
    double eta;
    // LM scalars
    double model_cost_change, cand_cost, step_norm2, x_norm2;
};

// Per-unknown finish of the problem build: column norms incl. regulariser rows, Jacobi scale, gradient.
//   c_j = w_g*cg[j] + (E_r, E_s, E_a analytic column norms);  s_j = free ? 1/(1+sqrt(c_j)) : 0
//   b_j = s_j * (w_g*bg[j] + regulariser gradient)
// (TrustRegionMinimizer jacobi_scaling + gradient; see oracle.cpp "jacobi scaling")
__global__ void __launch_bounds__(kThreads)
k_finish_problem(GridView g, RegView rv, SolveVecs sv, Shard sh, int64_t count, const double* __restrict__ type_w, const float* __restrict__ cam_acc, int fix_poses,
                 int fix_intr, int fix_dist, ReduceSite site /* [0] num params (free & colnorm>0), [1] x_norm^2 over those, [2] gmax^2 */,
                 const double* __restrict__ cam)
{
    pdl_prologue();
    const int64_t tbase = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) * 4;
    double acc[3] = {0.0, 0.0, 0.0};
#pragma unroll
    for (int e4 = 0; e4 < 4; ++e4)
    {
        const int64_t t = tbase + e4;
        if (t >= count) break;
        const int64_t j = sh.unknown(t, sv.n);
        const double wg = type_w[0], wr = type_w[1], ws = type_w[2], wa = type_w[3];
        double c = 0.0, grad = 0.0, xval = 0.0;
        bool free_ = false;
        const int64_t n = g.n;
        if (j < n)
        {
            const int64_t v = j;
            const uint8_t fl = rv.flags[v];
            free_ = fl & FL_FREE_SDF;
            c = wg * static_cast<double>(sv.cg[j]); grad = wg * static_cast<double>(sv.bg[j]);
            const bool hasEr = rv.use_er && (fl & FL_ACTIVE) && (fl & FL_RING);
            if (rv.use_er)
            {
                double cnt = hasEr ? 36.0 : 0.0, gl = hasEr ? -6.0 * rv.lap[v] : 0.0;
#pragma unroll
                for (int o = 0; o < 6; ++o)
                {
                    const int32_t nb = g.nbr[static_cast<int64_t>(o) * n + v];
                    if (nb >= 0)
                    {
                        const uint8_t fb = rv.flags[nb];
                        // nb's row contains v iff nb has an E_r row (its ring is valid, so v is valid)
                        if ((fb & FL_ACTIVE) && (fb & FL_RING)) { cnt += 1.0; gl += rv.lap[nb]; }
                    }
                }
                c += wr * cnt; grad += wr * gl;
            }
            if (rv.use_es && (fl & FL_ACTIVE) && (fl & FL_ES_JAC)) { c += ws; grad += ws * (g.sdf[v] - g.sdf0[v]); }
            xval = g.sdf[v];
        }
        else if (j < 2 * n)
        {
            const int64_t v = j - n;
            const uint8_t fl = rv.flags[v];
            free_ = fl & FL_FREE_ALB;
            c = wg * static_cast<double>(sv.cg[j]); grad = wg * static_cast<double>(sv.bg[j]);
            if (rv.use_ea)
            {
                const double av = g.albedo[v];
#pragma unroll
                for (int d = 0; d < 3; ++d)
                {
                    const float wp = rv.ea_w[static_cast<int64_t>(d) * n + v];
                    if (wp != 0.0f) { const int32_t b = g.nbr[static_cast<int64_t>(2 * d) * n + v]; c += wa * wp; grad += wa * wp * (av - g.albedo[b]); }
                    const int32_t m = g.nbr[static_cast<int64_t>(2 * d + 1) * n + v];
                    if (m >= 0)
                    {
                        const float wm = rv.ea_w[static_cast<int64_t>(d) * n + m];
                        if (wm != 0.0f) { c += wa * wm; grad += wa * wm * (av - g.albedo[m]); }
                    }
                }
            }
            xval = g.albedo[v];
        }
        else
        {
            const int64_t cidx = j - 2 * n;        // index into cam[]
            const CamAccLayout lay{sv.F};
            if (cidx < 6 * static_cast<int64_t>(sv.F))
            {
                const int f = static_cast<int>(cidx / 6), k = static_cast<int>(cidx - 6 * f);
                free_ = !fix_poses;
                grad = wg * static_cast<double>(cam_acc[lay.pose_stride() * f + k]);
                c = wg * static_cast<double>(cam_acc[lay.pose_stride() * f + 6 + k]);
            }
            else
            {
                const int k = static_cast<int>(cidx - 6 * static_cast<int64_t>(sv.F));
                free_ = (k < 4) ? !fix_intr : !fix_dist;
                grad = wg * static_cast<double>(cam_acc[lay.tail() + k]);
                c = wg * static_cast<double>(cam_acc[lay.tail() + 9 + k]);
            }
            xval = cam[cidx];
        }
        const double s = free_ ? 1.0 / (1.0 + sqrt(c)) : 0.0;
        sv.s[j] = static_cast<float>(s);
        sv.jtj[j] = static_cast<float>(s * s * c);
        sv.b[j] = static_cast<float>(s * grad);
        if (sh.owns_unknown(j, n))
        {
            if (free_ && c > 0.0) { acc[0] += 1.0; acc[1] += xval * xval; }
            if (free_) acc[2] += grad * grad;   // max-norm is taken on the host from the L2 bound (only used for the 1e-10 test)
        }
    }
    grid_reduce<3>(acc, site);
}

// LevenbergMarquardtStrategy: diag = clamp(colnorm^2(J'), min, max); D^2 = diag / radius
__device__ __forceinline__ float lm_diag(float jtj, float dmin, float dmax) { return fminf(fmaxf(jtj, dmin), dmax); }

// Block-Jacobi preconditioner blocks of the camera parameters (BlockJacobiPreconditioner + Invert):
// M_f = S G_f S * w_g + D^2, inverted by Cholesky in double.  One thread per block (F poses + intrinsics + distortion).
__device__ inline bool chol_inverse(int m, double* A /* m*m in, L out */, double* inv)
{
    for (int i = 0; i < m; ++i)
        for (int j = 0; j <= i; ++j)
        {
            double s = A[i * m + j];
            for (int k = 0; k < j; ++k) s -= A[i * m + k] * A[j * m + k];
            if (i == j) { if (!(s > 0.0)) return false; A[i * m + i] = sqrt(s); }
            else A[i * m + j] = s / A[j * m + j];
        }
    for (int c = 0; c < m; ++c)
    {
        double y[6], x[6];
        for (int i = 0; i < m; ++i)
        {
            double s = (i == c) ? 1.0 : 0.0;
            for (int k = 0; k < i; ++k) s -= A[i * m + k] * y[k];
            y[i] = s / A[i * m + i];
        }
        for (int i = m - 1; i >= 0; --i)
        {
            double s = y[i];
            for (int k = i + 1; k < m; ++k) s -= A[k * m + i] * x[k];
            x[i] = s / A[i * m + i];
        }
        for (int i = 0; i < m; ++i) inv[i * m + c] = x[i];
    }
    return true;
}

__global__ void k_cam_precond(SolveVecs sv, const float* __restrict__ cam_acc, const double* __restrict__ type_w, const CgCtl* __restrict__ ctl,
                              float dmin, float dmax, double* __restrict__ minv /* [F][36] + 16 + 25 */, int* __restrict__ fail)
{
    pdl_prologue();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int F = sv.F;
    if (t >= F + 2) return;
    const CamAccLayout lay{F};
    const double wg = type_w[0];
    const double inv_radius = ctl->inv_radius;
    int m; const float* tri; int64_t base; double* out;
    if (t < F) { m = 6; tri = cam_acc + lay.pose_stride() * t + 12; base = 2 * sv.n + 6 * static_cast<int64_t>(t); out = minv + 36 * static_cast<size_t>(t); }
    else if (t == F) { m = 4; tri = cam_acc + lay.tail() + 18; base = 2 * sv.n + 6 * static_cast<int64_t>(F); out = minv + 36 * static_cast<size_t>(F); }
    else { m = 5; tri = cam_acc + lay.tail() + 18 + 10; base = 2 * sv.n + 6 * static_cast<int64_t>(F) + 4; out = minv + 36 * static_cast<size_t>(F) + 16; }
    double A[36];
    int k = 0;
    for (int r = 0; r < m; ++r)
        for (int c = r; c < m; ++c)
        {
            const double val = wg * static_cast<double>(tri[k++]) * static_cast<double>(sv.s[base + r]) * static_cast<double>(sv.s[base + c]);
            A[r * m + c] = val; A[c * m + r] = val;
        }
    for (int r = 0; r < m; ++r) A[r * m + r] += static_cast<double>(lm_diag(sv.jtj[base + r], dmin, dmax)) * inv_radius;
    double inv[36];
    if (!chol_inverse(m, A, inv)) { atomicExch(fail, 1); for (int i = 0; i < m * m; ++i) inv[i] = 0.0; }
    for (int i = 0; i < m * m; ++i) out[i] = inv[i];
}

// ----------------------------------------------------------------------------------------------
// k5: the CGNR operator  q = J'^T (J' p) + D^2 p   (CgnrLinearOperator::RightMultiply), split in
//   k_eg_apply   E_g rows: one pass over J, fused J p and J^T (.) with atomics into qg; also the E_r row values of the input vector
//   k_op_post    regulariser rows (gather form) + D^2 + Jacobi scale, p.q partials
// ----------------------------------------------------------------------------------------------
enum { APPLY_CG = 0, APPLY_MODEL = 1 };


// k5: the E_g part of the CGNR operator.  One thread per active voxel; streams the K raw J rows of the voxel once
// (column-major J: every load of a warp is one full 128 B line).
//   u_k = J_k . ps          (ps = s o p, the Jacobi-scaled input)
//   APPLY_CG   : qg[cols] += sum_k w_k u_k J_k ; partial p.q += w_k u_k^2
//       voxel columns          : per-thread sums over the K rows, one global atomic per column per voxel
//       intrinsics/distortion  : per-thread sums, one warp reduce-scatter at the end
//       pose columns           : the K contributions of a thread (6 floats each) are parked in shared memory; after the row
//                                loop the warp walks over the DISTINCT frames among all of its 32 x K rows (typically 6-10),
//                                and for each does one 6-value butterfly all-reduce -> 6 shared-memory atomics.
//                                (A first version reduced per row slot: ~20 passes per warp, 49 % of the kernel's
//                                instructions were shuffle/select traffic; profiles/r01_summary.md.)
//   APPLY_MODEL: partial model_cost_change += -w_k u_k (r_k + u_k/2)          (TrustRegionMinimizer::ComputeTrustRegionStep)
// Contributions are added in double.  A double sum of B float addends is exact, and so independent of the atomics' order, when
// all addends of one entry lie within about 2^(29 - log2 B) of each other; where they do not, only the final rounding to float
// hides the order.  Measured: the full C3 scene (1.31 M active voxels, 5101 blocks, 200 frames) gives bit-identical results from
// run to run over three GN iterations (tests/test_gpu_round2.py::test_c3_run_to_run_bit_identical).
// (A bulk-async / mbarrier staged variant was measured slower: the kernel is issue-bound, not latency-bound.)
template <int MODE>
__global__ void __launch_bounds__(kThreads)
k_eg_apply(GridView g, EgRows rows, RegView rv, SolveVecs sv, const float* __restrict__ ps, const CgCtl* __restrict__ ctl, int respect_done, ReduceSite site)
{
    pdl_prologue();
    extern __shared__ double s_dyn_d[];  // [6F + 9] camera accumulators (double) | [K][6][kThreads] parked pose contributions (float)
    if (respect_done && ctl->done) return;
    const int ncam = 6 * sv.F + 9;
    double* s_cam = s_dyn_d;
    float* s_jp = reinterpret_cast<float*>(s_dyn_d + ((ncam + 15) & ~15));
    if (MODE == APPLY_CG)
    {
        for (int i = threadIdx.x; i < ncam; i += blockDim.x) s_cam[i] = 0.0;
        __syncthreads();
    }
    const int tid = threadIdx.x, lane = tid & 31;
    const int a = blockIdx.x * blockDim.x + tid;
    const bool in_range = a < rows.n_active;
    const int64_t n = g.n;
    const size_t S = static_cast<size_t>(rows.K) * rows.stride;
    double acc[1] = {0.0};
    int fk[I3D_MAX_OBS];
    bool any = false;
#pragma unroll
    for (int k = 0; k < I3D_MAX_OBS; ++k)
    {
        fk[k] = (in_range && k < rows.K) ? rows.row_frame[static_cast<size_t>(k) * rows.stride + a] : -1;
        any = any || (fk[k] >= 0);
    }
    float pv[14], out[14], pt[9], tail[9];
#pragma unroll
    for (int m = 0; m < 14; ++m) { pv[m] = 0.0f; out[m] = 0.0f; }
#pragma unroll
    for (int m = 0; m < 9; ++m) { pt[m] = ps[2 * n + 6 * static_cast<int64_t>(sv.F) + m]; tail[m] = 0.0f; }
    uint32_t idx[14];
    // E_r row of this voxel (rows exist exactly on the active voxels with a valid 6-ring, i.e. a subset of this kernel's voxels): its
    // value for the input vector, consumed by k_op_partial in gather form.  tr is zeroed once per GN iteration, so only these voxels
    // ever write it.  (Round 1 ran a separate kernel over all owned voxels for this: one launch per operator application.)
    if (in_range && rv.use_er)
    {
        const int64_t v = rows.act[a];
        if (rv.flags[v] & FL_RING)
        {
            float t = -6.0f * ps[v];
#pragma unroll
            for (int o = 0; o < 6; ++o) t += ps[g.nbr[static_cast<int64_t>(o) * n + v]];
            sv.tr[v] = t;
        }
    }
    if (any)
    {
        const int64_t v = rows.act[a];
        const uint32_t xp = g.nbr[NB_XP * n + v], yp = g.nbr[NB_YP * n + v], zp = g.nbr[NB_ZP * n + v];
        const uint32_t un = static_cast<uint32_t>(n);
        idx[0] = static_cast<uint32_t>(v); idx[1] = yp; idx[2] = g.nbr[NB_Y2 * n + v]; idx[3] = g.nbr[NB_YZ * n + v]; idx[4] = zp; idx[5] = g.nbr[NB_Z2 * n + v];
        idx[6] = xp; idx[7] = g.nbr[NB_XY * n + v]; idx[8] = g.nbr[NB_XZ * n + v]; idx[9] = g.nbr[NB_X2 * n + v];
        idx[10] = un + idx[0]; idx[11] = un + xp; idx[12] = un + yp; idx[13] = un + zp;
#pragma unroll
        for (int m = 0; m < 14; ++m) pv[m] = ps[idx[m]];
    }
#pragma unroll
    for (int k = 0; k < I3D_MAX_OBS; ++k)
    {
        if (k >= rows.K) break;
        const int f = fk[k];
        if (f >= 0)
        {
            const size_t slot = static_cast<size_t>(k) * rows.stride + a;
            const float* __restrict__ jc = rows.J + slot;
            float jr[29];
#pragma unroll
            for (int m = 0; m < 29; ++m) jr[m] = __ldcs(jc + static_cast<size_t>(m) * S);
            const float w = rows.row_w[slot];
            const float* pp = ps + 2 * n + 6 * static_cast<int64_t>(f);
            // four independent partial sums instead of one 29-long dependent FMA chain
            float u0 = 0.0f, u1 = 0.0f, u2 = 0.0f, u3 = 0.0f;
#pragma unroll
            for (int m = 0; m < 12; m += 4) { u0 += jr[m] * pv[m]; u1 += jr[m + 1] * pv[m + 1]; u2 += jr[m + 2] * pv[m + 2]; u3 += jr[m + 3] * pv[m + 3]; }
            u0 += jr[12] * pv[12]; u1 += jr[13] * pv[13];
#pragma unroll
            for (int c = 0; c < 6; c += 2) { u2 += jr[14 + c] * pp[c]; u3 += jr[15 + c] * pp[c + 1]; }
#pragma unroll
            for (int m = 0; m < 8; m += 4) { u0 += jr[20 + m] * pt[m]; u1 += jr[21 + m] * pt[m + 1]; u2 += jr[22 + m] * pt[m + 2]; u3 += jr[23 + m] * pt[m + 3]; }
            u0 += jr[28] * pt[8];
            const float u = (u0 + u1) + (u2 + u3);
            if (MODE == APPLY_CG)
            {
                const float wu = w * u;
                acc[0] += static_cast<double>(wu) * static_cast<double>(u);
#pragma unroll
                for (int m = 0; m < 14; ++m) out[m] += wu * jr[m];
#pragma unroll
                for (int c = 0; c < 6; ++c) s_jp[(k * 6 + c) * kThreads + tid] = wu * jr[14 + c];
#pragma unroll
                for (int m = 0; m < 9; ++m) tail[m] += wu * jr[20 + m];
            }
            else
            {
                const double r = rows.row_res[slot];
                acc[0] -= static_cast<double>(w) * static_cast<double>(u) * (r + 0.5 * static_cast<double>(u));
            }
        }
    }
    if (MODE == APPLY_CG)
    {
        // ---- pose columns: walk over the distinct frames of the warp's 32 x K rows
        // (measured alternative, slower: reducing a slot straight from registers when all 32 rows of the warp share its frame and
        // parking only mixed slots — 0.305 vs 0.289 ms per launch at C3: the uniformity test costs more than the walk it saves)
        unsigned todo = 0u;                       // bit k: slot k of this lane still has to be added
#pragma unroll
        for (int k = 0; k < I3D_MAX_OBS; ++k) if (fk[k] >= 0) todo |= 1u << k;
        while (true)
        {
            const unsigned pending = __ballot_sync(0xffffffffu, todo != 0u);
            if (pending == 0u) break;
            const int leader = __ffs(pending) - 1;
            const int mine_f = (todo != 0u) ? fk_select(fk, __ffs(todo) - 1) : -1;
            const int f0 = __shfl_sync(0xffffffffu, mine_f, leader);
            float r8[8] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
            for (int k = 0; k < I3D_MAX_OBS; ++k)
            {
                if (k >= rows.K) break;
                if (((todo >> k) & 1u) && fk[k] == f0)
                {
#pragma unroll
                    for (int c = 0; c < 6; ++c) r8[c] = s_jp[(k * 6 + c) * kThreads + tid];
                    todo &= ~(1u << k);
                }
            }
            // 8 -> 1 value per lane in three halving exchanges (offsets 16, 8, 4), then an all-reduce over the remaining two
            // lane bits: 4 + 2 + 1 + 1 + 1 = 9 shuffles (a plain all-reduce of the 6 values needs 30)
            rs_step<4, 16, 8>(r8, lane);
            rs_step<2, 8, 8>(r8, lane);
            rs_step<1, 4, 8>(r8, lane);
            float val = r8[0];
            val += __shfl_xor_sync(0xffffffffu, val, 2);
            val += __shfl_xor_sync(0xffffffffu, val, 1);
            const int id = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
            if ((lane & 3) == 0 && id < 6 && val != 0.0f) atomicAdd(s_cam + 6 * f0 + id, static_cast<double>(val));
        }
        if (any)
        {
#pragma unroll
            for (int m = 0; m < 14; ++m) atomicAdd(sv.qgd + idx[m], static_cast<double>(out[m]));
        }
        {
            float vv[32];
#pragma unroll
            for (int m = 0; m < 9; ++m) vv[m] = tail[m];
#pragma unroll
            for (int m = 9; m < 32; ++m) vv[m] = 0.0f;
            warp_reduce_scatter<32>(vv, lane);
            if (lane < 9 && vv[0] != 0.0f) atomicAdd(s_cam + 6 * sv.F + lane, static_cast<double>(vv[0]));
        }
        __syncthreads();
        // block partial rounded to float, then summed over blocks in double: exact while the partials of one entry stay within
        // about 2^(29 - log2 B) of each other, B = contributing blocks (see the kernel's comment for what was measured)
        for (int i = tid; i < ncam; i += blockDim.x) { const float vv = static_cast<float>(s_cam[i]); if (vv != 0.0f) atomicAdd(sv.qgd + 2 * sv.n + i, static_cast<double>(vv)); }
    }
    grid_reduce<1>(acc, site);
}

// ---- scalar epilogues of the PCG iteration (ConjugateGradientsSolver::Solve restated).  Single GPU: run by the last
// block of the producing kernel; multi GPU: run by k_epilogue after the allreduce of the partial sums.
__device__ __forceinline__ void epilogue_operator(CgCtl* ctl, double total, int mode, int is_cg_iteration)
{
    if (mode == APPLY_MODEL) { ctl->model_cost_change = total; return; }
    if (!is_cg_iteration) return;
    ctl->pq = total;
    if (total <= 0.0 || isinf(total)) { ctl->done = 1; ctl->status = 2; ctl->it += 1; ctl->alpha = 0.0; }
    else
    {
        const double alpha = ctl->rho / total;
        if (isinf(alpha)) { ctl->done = 1; ctl->status = 1; ctl->alpha = 0.0; }
        else ctl->alpha = alpha;
    }
}

__device__ __forceinline__ void epilogue_update(CgCtl* ctl, double rho_new, double Q1, double xd2x, bool init)
{
    if (init)
    {
        ctl->it = 0; ctl->Q0 = 0.0; ctl->Q1 = 0.0; ctl->zeta = 0.0; ctl->status = 0; ctl->alpha = 0.0; ctl->pq = 0.0; ctl->xd2x = 0.0;
        ctl->rho = rho_new; ctl->last_rho = 1.0; ctl->beta = 0.0;
        // |b| == 0  <=>  rho == 0 for an SPD preconditioner: ceres returns x = 0 ("Convergence. |b| = 0.")
        if (rho_new == 0.0) { ctl->done = 1; ctl->status = 0; }
        else if (!isfinite(rho_new)) { ctl->done = 1; ctl->status = 1; }
        else ctl->done = ctl->halt ? 1 : 0;
        return;
    }
    const int it = ctl->it + 1;
    ctl->it = it;
    const double zeta = it * (Q1 - ctl->Q0) / Q1;
    ctl->Q1 = Q1; ctl->zeta = zeta; ctl->xd2x = xd2x;
    bool stop = false;
    if (ctl->forced_iterations > 0) { if (it >= ctl->forced_iterations) { stop = true; ctl->status = 0; } }
    else
    {
        if (zeta < ctl->eta && it >= ctl->min_iterations) { stop = true; ctl->status = 0; }
        else if (it >= ctl->max_iterations) { stop = true; ctl->status = 3; }
    }
    ctl->Q0 = Q1;
    if (!stop)
    {
        ctl->last_rho = ctl->rho; ctl->rho = rho_new;
        const double beta = rho_new / ctl->last_rho;
        if (rho_new == 0.0 || !isfinite(rho_new) || beta == 0.0 || !isfinite(beta)) { stop = true; ctl->status = 1; }
        ctl->beta = beta;
    }
    if (stop) ctl->done = 1;
}

enum { EPI_OPERATOR_CG = 0, EPI_OPERATOR_NOCG = 1, EPI_MODEL = 2, EPI_UPDATE = 3, EPI_UPDATE_INIT = 4 };
// multi-GPU: scalars[] holds the ALLREDUCED sums
__global__ void k_epilogue(CgCtl* __restrict__ ctl, const double* __restrict__ scalars, int kind, int respect_done)
{
    pdl_prologue();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (respect_done && kind != EPI_UPDATE_INIT && ctl->done) return;
    if (kind == EPI_OPERATOR_CG) epilogue_operator(ctl, scalars[0], APPLY_CG, 1);
    else if (kind == EPI_MODEL) epilogue_operator(ctl, scalars[0], APPLY_MODEL, 0);
    else if (kind == EPI_UPDATE) epilogue_update(ctl, scalars[0], scalars[1], scalars[2], false);
    else if (kind == EPI_UPDATE_INIT) epilogue_update(ctl, scalars[0], scalars[1], scalars[2], true);
}

// Per-unknown part of the operator: adds the regulariser rows OWNED by this rank (gather form) into qg, in place:
//     qg[j] += qgd[j] (k_eg_apply's E_g part, rounded once; qgd is cleared) + sum over owned E_r / E_s / E_a rows touching j
//     (raw, Jacobi scale applied by the consumer)
// The operator output  q_j = s_j * qg_j(total) + D_j^2 p_j  is never materialised: k_cg_update forms it on the fly.
// MODE APPLY_CG   : partial p.q += (owned regulariser rows)^2 + D^2 p^2 (owned unknowns); last block: alpha = rho / pq.
// MODE APPLY_MODEL: partial model_cost_change of the owned regulariser rows (qg untouched).
template <int MODE, int VEC>
__global__ void __launch_bounds__(kThreads)
k_op_partial(GridView g, RegView rv, SolveVecs sv, Shard sh, int64_t count, const float* __restrict__ pin, const float* __restrict__ ps,
             const double* __restrict__ type_w, float dmin, float dmax, CgCtl* __restrict__ ctl, int respect_done,
             ReduceSite site, const double* __restrict__ eg_partial /* site.out of k_eg_apply */, int is_cg_iteration)
{
    pdl_prologue();
    if (respect_done && ctl->done) return;
    const int64_t tbase = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) * VEC;
    double acc[1] = {0.0};
    const int64_t n = g.n;
    const float wr = static_cast<float>(type_w[1]), ws = static_cast<float>(type_w[2]), wa = static_cast<float>(type_w[3]);
    const float inv_radius = static_cast<float>(ctl->inv_radius);
    // VEC consecutive unknowns per thread (unrolled: the gathers of the VEC elements are independent and overlap)
    float regs[VEC]; int64_t js[VEC];
#pragma unroll
    for (int e = 0; e < VEC; ++e) { regs[e] = 0.0f; js[e] = 0; }
#pragma unroll
    for (int e = 0; e < VEC; ++e)
    {
        const int64_t t = tbase + e;
        if (t >= count) break;
        const int64_t j = sh.unknown(t, sv.n);
        float reg = 0.0f;
        if (j < n)
        {
            const int64_t v = j;
            const uint8_t fl = rv.flags[v];
            const bool own = sh.owns_voxel(v);
            if (rv.use_er)
            {
                const float t0 = own ? sv.tr[v] : 0.0f;
                float tt = -6.0f * t0;
#pragma unroll
                for (int o = 0; o < 6; ++o) { const int32_t nb = g.nbr[static_cast<int64_t>(o) * n + v]; if (nb >= 0 && sh.owns_voxel(nb)) tt += sv.tr[nb]; }
                reg += wr * tt;
                if (MODE == APPLY_CG) acc[0] += static_cast<double>(wr) * t0 * t0;
                else if (own) acc[0] -= static_cast<double>(wr) * t0 * (rv.lap[v] + 0.5 * static_cast<double>(t0));
            }
            if (rv.use_es && own && (fl & FL_ACTIVE) && (fl & FL_ES_JAC))
            {
                const float u = ps[v];
                reg += ws * u;
                if (MODE == APPLY_CG) acc[0] += static_cast<double>(ws) * u * u;
                else acc[0] -= static_cast<double>(ws) * u * ((g.sdf[v] - g.sdf0[v]) + 0.5 * static_cast<double>(u));
            }
        }
        else if (j < 2 * n)
        {
            const int64_t v = j - n;
            if (rv.use_ea)
            {
                const float pa = ps[j];
                const bool own = sh.owns_voxel(v);
#pragma unroll
                for (int d = 0; d < 3; ++d)
                {
                    // the pair {v, v + e_d} is stored at (d, v): it belongs to the rank that owns v
                    const float wp = own ? rv.ea_w[static_cast<int64_t>(d) * n + v] : 0.0f;
                    if (wp != 0.0f)
                    {
                        const int32_t b = g.nbr[static_cast<int64_t>(2 * d) * n + v];
                        const float du = pa - ps[n + b];
                        reg += wa * wp * du;
                        if (MODE == APPLY_CG) acc[0] += static_cast<double>(wa) * wp * du * du;
                        else acc[0] -= static_cast<double>(wa) * wp * du * ((g.albedo[v] - g.albedo[b]) + 0.5 * static_cast<double>(du));
                    }
                    const int32_t m = g.nbr[static_cast<int64_t>(2 * d + 1) * n + v];
                    if (m >= 0 && sh.owns_voxel(m))
                    {
                        const float wm = rv.ea_w[static_cast<int64_t>(d) * n + m];
                        if (wm != 0.0f) reg += wa * wm * (pa - ps[n + m]);
                    }
                }
            }
        }
        if (MODE == APPLY_CG)
        {
            regs[e] = reg; js[e] = j;       // the read-modify-write of qg is deferred so that the gathers of the next element can start
            if (sh.owns_unknown(j, n))
            {
                const float pj = pin[j];
                const float d2 = lm_diag(sv.jtj[j], dmin, dmax) * inv_radius;
                acc[0] += static_cast<double>(d2) * pj * pj;
            }
        }
    }
    if (MODE == APPLY_CG)
    {
#pragma unroll
        for (int e = 0; e < VEC; ++e)
        {
            if (tbase + e >= count) break;
            const double eg = sv.qgd[js[e]];
            if (eg != 0.0) sv.qgd[js[e]] = 0.0;
            const float add = static_cast<float>(eg) + regs[e];
            if (add != 0.0f) sv.qg[js[e]] += add;
        }
    }
    if (grid_reduce<1>(acc, site) && threadIdx.x == 0)
    {
        // fold the E_g partial in so that site.out[0] is this rank's complete partial sum
        const double total = site.out[0] + eg_partial[0];
        site.out[0] = total;
        if (!sh.defer) epilogue_operator(ctl, total, MODE, is_cg_iteration);
    }
}

// x += alpha p (first half of an exact-residual refresh iteration)
__global__ void k_x_update(SolveVecs sv, Shard sh, int64_t count, const CgCtl* __restrict__ ctl)
{
    pdl_prologue();
    if (ctl->done) return;
    const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (t >= count) return;
    const int64_t j = sh.unknown(t, sv.n);
    sv.x[j] += static_cast<float>(ctl->alpha) * sv.p[j];
}

// out = sign * s o v (for the exact-residual refresh and the model evaluation)
__global__ void k_scale_vec(SolveVecs sv, Shard sh, int64_t count, const float* __restrict__ v, float sign, float* __restrict__ out,
                            const CgCtl* __restrict__ ctl, int respect_done)
{
    pdl_prologue();
    if (respect_done && ctl->done) return;
    const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (t >= count) return;
    const int64_t j = sh.unknown(t, sv.n);
    out[j] = sign * sv.s[j] * v[j];
}

// 4 consecutive floats with one 16 B access (single-GPU identity layout only; all vectors are cudaMalloc-aligned)
__device__ __forceinline__ void ld4(const float* __restrict__ p, int64_t j, float (&v)[4])
{
    const float4 t = *reinterpret_cast<const float4*>(p + j);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void st4(float* __restrict__ p, int64_t j, const float (&v)[4])
{
    *reinterpret_cast<float4*>(p + j) = make_float4(v[0], v[1], v[2], v[3]);
}

// x += alpha p ; r -= alpha q (or r = b - A x when refresh) ; z = M^-1 r ; partials rho = r.z, 2Q = -x.(b + r), x.D^2 x.
// The operator output is formed on the fly from the accumulated qg:  q_j = s_j qg_j + D_j^2 v_j  (v = p, or x when
// refreshing), and qg_j is reset to zero for the next application.
// INIT: x = 0, r = b.  Epilogue: Q-based termination test and beta for the next iteration.
// The first F + 2 threads handle one camera block each (serial 6x6 work, scheduled first so that it overlaps the streaming
// part); the remaining threads handle the voxel unknowns: VEC = 4 consecutive unknowns per thread with 16 B accesses in the
// single-GPU identity layout, VEC = 1 through the held list when sharded.
template <bool INIT, int VEC>
__global__ void __launch_bounds__(kThreads)
k_cg_update(SolveVecs sv, Shard sh, const double* __restrict__ minv, float dmin, float dmax, CgCtl* __restrict__ ctl, int refresh, ReduceSite site)
{
    pdl_prologue();
    if (!INIT && ctl->done) return;
    const int64_t t0 = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    const int64_t ncb = sv.F + 2;
    const int64_t n2 = 2 * sv.n;
    const int64_t nvox = sh.held_voxel_unknowns();
    const bool is_cam = t0 < ncb;
    double acc[3] = {0.0, 0.0, 0.0};      // rho = r.z, 2Q = -x.(b + r), x.D^2 x
    const float alpha = INIT ? 0.0f : static_cast<float>(ctl->alpha);
    const float inv_radius = static_cast<float>(ctl->inv_radius);
    if (!is_cam)
    {
        const int64_t e0 = (t0 - ncb) * VEC;
        int64_t j0 = 0;
        if (VEC == 4 && sh.vec4(e0, sv.n, &j0))
        {
            float bj[4], jt[4], sj[4], qg[4], vj[4], xo[4], ro[4], xn[4], rn[4], zn[4];
            ld4(sv.b, j0, bj); ld4(sv.jtj, j0, jt);
            if (!INIT)
            {
                ld4(sv.s, j0, sj); ld4(sv.qg, j0, qg); ld4(sv.x, j0, xo);
                if (refresh) { for (int i = 0; i < 4; ++i) vj[i] = xo[i]; } else { ld4(sv.p, j0, vj); ld4(sv.r, j0, ro); }
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
            {
                const float d2 = lm_diag(jt[i], dmin, dmax) * inv_radius;
                if (INIT) { xn[i] = 0.0f; rn[i] = bj[i]; }
                else
                {
                    const float qj = sj[i] * qg[i] + d2 * vj[i];
                    xn[i] = refresh ? xo[i] : (xo[i] + alpha * vj[i]);
                    rn[i] = refresh ? (bj[i] - qj) : (ro[i] - alpha * qj);
                }
                zn[i] = rn[i] / (jt[i] + d2);
                if (sh.owns_unknown(j0 + i, sv.n))
                {
                    acc[0] += static_cast<double>(rn[i]) * zn[i];
                    acc[1] -= static_cast<double>(xn[i]) * (static_cast<double>(bj[i]) + rn[i]);
                    acc[2] += static_cast<double>(d2) * xn[i] * xn[i];
                }
            }
            st4(sv.x, j0, xn); st4(sv.r, j0, rn); st4(sv.z, j0, zn);
            if (!INIT) { const float zero[4] = {0.0f, 0.0f, 0.0f, 0.0f}; st4(sv.qg, j0, zero); }
        }
        else
        {
#pragma unroll 1
            for (int64_t t = e0; t < e0 + VEC && t < nvox; ++t)
            {
                const int64_t j = sh.unknown(t, sv.n);
                const float bj = sv.b[j];
                const float jt = sv.jtj[j];
                const float d2 = lm_diag(jt, dmin, dmax) * inv_radius;
                float xj, rj;
                if (INIT) { xj = 0.0f; rj = bj; }
                else
                {
                    const float vj = refresh ? sv.x[j] : sv.p[j];
                    const float qj = sv.s[j] * sv.qg[j] + d2 * vj;
                    sv.qg[j] = 0.0f;
                    // refresh: x was already advanced by k_x_update and q = A x (exact residual, every residual_reset_period iterations)
                    xj = refresh ? sv.x[j] : (sv.x[j] + alpha * vj);
                    rj = refresh ? (bj - qj) : (sv.r[j] - alpha * qj);
                }
                const float zj = rj / (jt + d2);
                sv.x[j] = xj; sv.r[j] = rj; sv.z[j] = zj;
                if (sh.owns_unknown(j, sv.n))
                {
                    acc[0] += static_cast<double>(rj) * zj;
                    acc[1] -= static_cast<double>(xj) * (static_cast<double>(bj) + rj);
                    acc[2] += static_cast<double>(d2) * xj * xj;
                }
            }
        }
    }
    else
    {
        const int blk = static_cast<int>(t0);
        int m; int64_t base; const double* Mi;
        if (blk < sv.F) { m = 6; base = n2 + 6 * static_cast<int64_t>(blk); Mi = minv + 36 * static_cast<size_t>(blk); }
        else if (blk == sv.F) { m = 4; base = n2 + 6 * static_cast<int64_t>(sv.F); Mi = minv + 36 * static_cast<size_t>(sv.F); }
        else { m = 5; base = n2 + 6 * static_cast<int64_t>(sv.F) + 4; Mi = minv + 36 * static_cast<size_t>(sv.F) + 16; }
        float rr[6];
        double a0 = 0.0, a1 = 0.0, a2 = 0.0;
        for (int k = 0; k < m; ++k)
        {
            const int64_t j = base + k;
            const float bj = sv.b[j];
            const float d2 = lm_diag(sv.jtj[j], dmin, dmax) * inv_radius;
            float xj, rj;
            if (INIT) { xj = 0.0f; rj = bj; }
            else
            {
                const float vj = refresh ? sv.x[j] : sv.p[j];
                const float qj = sv.s[j] * sv.qg[j] + d2 * vj;
                sv.qg[j] = 0.0f;
                xj = refresh ? sv.x[j] : (sv.x[j] + alpha * vj);
                rj = refresh ? (bj - qj) : (sv.r[j] - alpha * qj);
            }
            sv.x[j] = xj; sv.r[j] = rj; rr[k] = rj;
            a1 -= static_cast<double>(xj) * (static_cast<double>(bj) + rj);
            a2 += static_cast<double>(d2) * xj * xj;
        }
        for (int i = 0; i < m; ++i)
        {
            double ssum = 0.0;
            for (int k = 0; k < m; ++k) ssum += Mi[i * m + k] * static_cast<double>(rr[k]);
            sv.z[base + i] = static_cast<float>(ssum);
            a0 += static_cast<double>(rr[i]) * ssum;
        }
        if (sh.cam_owner) { acc[0] = a0; acc[1] = a1; acc[2] = a2; }
    }
    if (grid_reduce<3>(acc, site) && threadIdx.x == 0 && !sh.defer) epilogue_update(ctl, site.out[0], site.out[1], site.out[2], INIT);
}

// p = z + beta p ; ps = s o p over the unknowns this rank holds, 4 per thread with 16 B accesses where the group is aligned
__global__ void __launch_bounds__(kThreads)
k_cg_dir4(SolveVecs sv, Shard sh, int64_t count, const CgCtl* __restrict__ ctl)
{
    pdl_prologue();
    if (ctl->done) return;
    const int64_t e0 = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) * 4;
    if (e0 >= count) return;
    const float beta = static_cast<float>(ctl->beta);
    int64_t j0 = 0;
    if (sh.vec4(e0, sv.n, &j0))
    {
        float z[4], p[4], s4[4], ps[4];
        ld4(sv.z, j0, z); ld4(sv.p, j0, p); ld4(sv.s, j0, s4);
#pragma unroll
        for (int i = 0; i < 4; ++i) { p[i] = (beta == 0.0f) ? z[i] : z[i] + beta * p[i]; ps[i] = s4[i] * p[i]; }      // first iteration: p may hold anything
        st4(sv.p, j0, p); st4(sv.ps, j0, ps);
    }
    else
        for (int64_t t = e0; t < e0 + 4 && t < count; ++t)
        {
            const int64_t j = sh.unknown(t, sv.n);
            const float p = (beta == 0.0f) ? sv.z[j] : sv.z[j] + beta * sv.p[j];
            sv.p[j] = p; sv.ps[j] = sv.s[j] * p;
        }
}

// ---- multi-GPU exchange buffers ---------------------------------------------------------------------------------
// xbuf (double) = [ v0 at shared unknowns | v1 at shared unknowns (optional) | extra floats | extra doubles ]
struct ShareView
{
    int64_t n_shared;
    const int32_t* slist;    // shared unknown indices (ascending), identical on every rank
    const uint8_t* held;     // [2n] this rank holds the unknown (contributes / consumes); others contribute 0
};

__global__ void k_pack(ShareView sh, const float* __restrict__ v0, const float* __restrict__ v1, const float* __restrict__ extra_f, int n_extra_f,
                       const double* __restrict__ extra_d, int n_extra_d, double* __restrict__ xbuf, const CgCtl* __restrict__ ctl, int respect_done)
{
    pdl_prologue();
    if (respect_done && ctl->done) return;
    const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    const int64_t nv = v1 ? 2 : 1;
    if (t < sh.n_shared)
    {
        const int32_t j = sh.slist[t];
        const bool h = sh.held[j] != 0;
        xbuf[t] = h ? static_cast<double>(v0[j]) : 0.0;
        if (v1) xbuf[sh.n_shared + t] = h ? static_cast<double>(v1[j]) : 0.0;
    }
    else if (t < sh.n_shared + n_extra_f) xbuf[nv * sh.n_shared + (t - sh.n_shared)] = static_cast<double>(extra_f[t - sh.n_shared]);
    else if (t < sh.n_shared + n_extra_f + n_extra_d) xbuf[nv * sh.n_shared + (t - sh.n_shared)] = extra_d[t - sh.n_shared - n_extra_f];
}

__global__ void k_unpack(ShareView sh, float* __restrict__ v0, float* __restrict__ v1, float* __restrict__ extra_f, int n_extra_f,
                         double* __restrict__ extra_d, int n_extra_d, const double* __restrict__ xbuf, const CgCtl* __restrict__ ctl, int respect_done)
{
    pdl_prologue();
    if (respect_done && ctl->done) return;
    const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    const int64_t nv = v1 ? 2 : 1;
    if (t < sh.n_shared)
    {
        const int32_t j = sh.slist[t];
        if (sh.held[j]) { v0[j] = static_cast<float>(xbuf[t]); if (v1) v1[j] = static_cast<float>(xbuf[sh.n_shared + t]); }
    }
    else if (t < sh.n_shared + n_extra_f) extra_f[t - sh.n_shared] = static_cast<float>(xbuf[nv * sh.n_shared + (t - sh.n_shared)]);
    else if (t < sh.n_shared + n_extra_f + n_extra_d) extra_d[t - sh.n_shared - n_extra_f] = xbuf[nv * sh.n_shared + (t - sh.n_shared)];
}

// ---- peer-memory exchange over NVLink (replaces the packed ncclAllReduce inside the PCG loop) ------------------------------
// Every rank owns a MAILBOX in its own HBM, mapped into every peer with CUDA IPC:
//     flags[world]        flags[r] = sequence number of the last exchange rank r has published (written REMOTELY by rank r)
//     data[2][cap]        this rank's packed partial sums of exchange `seq`, in buffer seq & 1 (written locally by k_pack)
// One exchange = k_pack (local) + k_xchg_pull: publish `seq` into every peer's flag array (one remote 4-byte store each),
// wait until every peer has published `seq` (spin on LOCAL memory), then PULL the peers' buffers (coalesced remote loads
// over NVLink), add them in rank order — every rank adds the same numbers in the same order, so all ranks end with bit-identical
// sums (what the solver needs: identical vector updates on the unknowns several ranks hold) — and unpack.
// Two buffers suffice: a rank publishes seq+1 only after its own pull of seq has finished (stream order), so once a rank has
// seen everybody's seq+1 flags nobody reads buffer (seq & 1) any more and it may be overwritten for seq+2.  The handshake is
// executed even when the PCG has converged (`done`): it is what keeps the ranks in lock step.
struct P2PView
{
    int rank, world;
    double* const* peer_data;          // [world] base of every rank's data region (own entry = local pointer)
    unsigned int* const* peer_flags;   // [world] base of every rank's flag array
    size_t cap;                        // doubles per buffer
};

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p)
{
    unsigned int v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ double ld_peer_f64(const double* p)
{
    double v;
    asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");     // never served from a stale L1 line
    return v;
}

// publish + wait (every block waits: the pulls below may only start once every peer's buffer is complete)
__device__ __forceinline__ void p2p_handshake(const P2PView& pp, unsigned int seq)
{
    if (blockIdx.x == 0 && threadIdx.x < static_cast<unsigned>(pp.world) && static_cast<int>(threadIdx.x) != pp.rank)
    {
        __threadfence_system();
        st_release_sys(pp.peer_flags[threadIdx.x] + pp.rank, seq);
    }
    if (threadIdx.x < static_cast<unsigned>(pp.world) && static_cast<int>(threadIdx.x) != pp.rank)
    {
        const unsigned int* f = pp.peer_flags[pp.rank] + threadIdx.x;
        while (static_cast<int>(ld_acquire_sys(f) - seq) < 0) { }          // wrap-safe comparison
    }
    __syncthreads();
}

// the pull half of an exchange: same argument meaning as k_unpack; xbuf layout [v0 | v1 | extra floats | extra doubles]
__global__ void __launch_bounds__(kThreads)
k_xchg_pull(P2PView pp, unsigned int seq, ShareView sh, float* __restrict__ v0, float* __restrict__ v1, float* __restrict__ extra_f, int n_extra_f,
            double* __restrict__ extra_d, int n_extra_d, CgCtl* __restrict__ ctl, int respect_done, int epilogue_kind /* EPI_* consuming extra_d[0], or -1 */)
{
    pdl_prologue();
    p2p_handshake(pp, seq);
    if (respect_done && ctl->done) return;              // identical on every rank (ctl is replicated state)
    const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    const int64_t nv = v1 ? 2 : 1;
    const size_t off = static_cast<size_t>(seq & 1u) * pp.cap;
    if (t < sh.n_shared)
    {
        const int32_t j = sh.slist[t];
        if (sh.held[j])
        {
            double a = 0.0, b = 0.0;
            for (int r = 0; r < pp.world; ++r)
            {
                a += ld_peer_f64(pp.peer_data[r] + off + t);
                if (v1) b += ld_peer_f64(pp.peer_data[r] + off + sh.n_shared + t);
            }
            v0[j] = static_cast<float>(a);
            if (v1) v1[j] = static_cast<float>(b);
        }
    }
    else if (t < sh.n_shared + n_extra_f + n_extra_d)
    {
        const size_t idx = static_cast<size_t>(nv * sh.n_shared + (t - sh.n_shared));
        double a = 0.0;
        for (int r = 0; r < pp.world; ++r) a += ld_peer_f64(pp.peer_data[r] + off + idx);
        if (t < sh.n_shared + n_extra_f) extra_f[t - sh.n_shared] = static_cast<float>(a);
        else
        {
            extra_d[t - sh.n_shared - n_extra_f] = a;
            // the scalar epilogue of the operator (alpha = rho / p.q) by the one thread that just summed p.q.  It can only SET `done`
            // (p.q <= 0: the solve stops and this application is discarded), so blocks of this launch that read `done` later and skip
            // their unpacking are harmless.
            if (t == sh.n_shared + n_extra_f && epilogue_kind >= 0)
            {
                if (epilogue_kind == EPI_OPERATOR_CG) epilogue_operator(ctl, a, APPLY_CG, 1);
                else if (epilogue_kind == EPI_MODEL) epilogue_operator(ctl, a, APPLY_MODEL, 0);
            }
        }
    }
}

// all-reduce of a few doubles + the scalar epilogue that consumes them, in ONE single-warp launch (replaces a 2-double
// ncclAllReduce + k_epilogue per PCG iteration): lane r talks to rank r.
__global__ void k_xchg_scalars(P2PView pp, unsigned int seq, double* __restrict__ vals, int count /* <= 30 */, CgCtl* __restrict__ ctl, int kind, int respect_done)
{
    pdl_prologue();
    const int lane = threadIdx.x;
    double* mine = pp.peer_data[pp.rank] + static_cast<size_t>(seq & 1u) * pp.cap;
    if (lane < count) mine[lane] = vals[lane];
    __syncwarp();
    p2p_handshake(pp, seq);
    if (respect_done && kind != EPI_UPDATE_INIT && kind >= 0 && ctl->done) return;
    if (lane < count)
    {
        double a = 0.0;
        for (int r = 0; r < pp.world; ++r) a += ld_peer_f64(pp.peer_data[r] + static_cast<size_t>(seq & 1u) * pp.cap + lane);
        vals[lane] = a;
    }
    __syncwarp();
    if (lane == 0 && kind >= 0)
    {
        if (kind == EPI_OPERATOR_CG) epilogue_operator(ctl, vals[0], APPLY_CG, 1);
        else if (kind == EPI_MODEL) epilogue_operator(ctl, vals[0], APPLY_MODEL, 0);
        else if (kind == EPI_UPDATE) epilogue_update(ctl, vals[0], vals[1], vals[2], false);
        else if (kind == EPI_UPDATE_INIT) epilogue_update(ctl, vals[0], vals[1], vals[2], true);
    }
}

// marks the unknowns touched by the rows of the voxels this rank owns (static: depends on the grid topology only)
__global__ void k_touch(GridView g, Shard sh, uint8_t* __restrict__ touch /* [2n] */)
{
    const int64_t v = sh.own_begin + blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (v >= sh.own_end) return;
    const int64_t n = g.n;
    touch[v] = 1; touch[n + v] = 1;
#pragma unroll
    for (int o = 0; o < NB_COUNT; ++o)
    {
        const int32_t nb = g.nbr[static_cast<int64_t>(o) * n + v];
        if (nb >= 0) { touch[nb] = 1; if (o == NB_XP || o == NB_YP || o == NB_ZP) touch[n + nb] = 1; }
    }
}
// smallest index range containing [lo, hi) and every stencil neighbour of its voxels: out[0] = min, out[1] = max (inclusive)
__global__ void k_range_extend(GridView g, int64_t lo, int64_t hi, int* __restrict__ out)
{
    const int64_t v = lo + blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    int mn = INT_MAX, mx = -1;
    if (v < hi)
    {
        mn = mx = static_cast<int>(v);
#pragma unroll
        for (int o = 0; o < NB_COUNT; ++o)
        {
            const int32_t nb = g.nbr[static_cast<int64_t>(o) * g.n + v];
            if (nb >= 0) { mn = min(mn, nb); mx = max(mx, nb); }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
    if ((threadIdx.x & 31) == 0) { atomicMin(out, mn); atomicMax(out + 1, mx); }
}
// flag[j] = bit0: held by me (touch), bit1: shared (count >= 2)
__global__ void k_share_flags(int64_t n2, const uint8_t* __restrict__ touch, const uint8_t* __restrict__ count, uint8_t* __restrict__ flags)
{
    const int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (j >= n2) return;
    flags[j] = (touch[j] ? 1 : 0) | (count[j] >= 2 ? 2 : 0);
}
// keeps delta only at owned unknowns (before the full-state allreduce of an accepted step)
__global__ void k_mask_owned(SolveVecs sv, Shard sh, float* __restrict__ delta)
{
    pdl_prologue();
    const int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (j >= sv.U) return;
    if (!sh.owns_unknown(j, sv.n)) delta[j] = 0.0f;
}

// ----------------------------------------------------------------------------------------------
// LM candidate point and cost-only evaluation
// ----------------------------------------------------------------------------------------------
// delta = -s o x (undo Jacobi scaling, LM negation); candidate = state + delta; ||delta||^2 over owned unknowns.
// from_delta != 0: candidate = state + delta_out for ALL unknowns (delta_out already holds the allreduced full step).
__global__ void __launch_bounds__(kThreads)
k_candidate(GridView g, SolveVecs sv, Shard sh, int64_t count, int from_delta, const double* __restrict__ cam, double* __restrict__ c_sdf,
            double* __restrict__ c_alb, double* __restrict__ c_cam, float* __restrict__ delta_out, CgCtl* __restrict__ ctl, ReduceSite site)
{
    pdl_prologue();
    const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    double acc[1] = {0.0};
    if (t < count)
    {
        const int64_t j = from_delta ? t : sh.unknown(t, sv.n);
        float d;
        if (from_delta) d = delta_out[j];
        else { d = -sv.s[j] * sv.x[j]; delta_out[j] = d; }
        if (sh.owns_unknown(j, g.n)) acc[0] = static_cast<double>(d) * d;
        if (j < g.n) c_sdf[j] = g.sdf[j] + static_cast<double>(d);
        else if (j < 2 * g.n) c_alb[j - g.n] = g.albedo[j - g.n] + static_cast<double>(d);
        else c_cam[j - 2 * g.n] = cam[j - 2 * g.n] + static_cast<double>(d);
    }
    if (grid_reduce<1>(acc, site) && threadIdx.x == 0 && !sh.defer) ctl->step_norm2 = site.out[0];
}

// cost of the regulariser rows at an arbitrary state: out [0] sum r_Er^2 [1] sum r_Es^2 [2] sum w r_Ea^2
__global__ void __launch_bounds__(kThreads)
k_reg_cost(GridView g, RegView rv, Shard sh, const double* __restrict__ sdf, const double* __restrict__ alb, ReduceSite site)
{
    pdl_prologue();
    const int64_t v = sh.own_begin + blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    double acc[3] = {0.0, 0.0, 0.0};
    if (v < sh.own_end)
    {
        const uint8_t fl = rv.flags[v];
        const bool active = fl & FL_ACTIVE, ring = fl & FL_RING;
        if (rv.use_er && active && ring)
        {
            const double c = sdf[v];
            const double xp = sdf[g.nbr[NB_XP * g.n + v]], xm = sdf[g.nbr[NB_XM * g.n + v]];
            const double yp = sdf[g.nbr[NB_YP * g.n + v]], ym = sdf[g.nbr[NB_YM * g.n + v]];
            const double zp = sdf[g.nbr[NB_ZP * g.n + v]], zm = sdf[g.nbr[NB_ZM * g.n + v]];
            const double lap = ((xp + xm - 2.0 * c) + (yp + ym - 2.0 * c)) + (zp + zm - 2.0 * c);
            acc[0] = lap * lap;
        }
        if (rv.use_es && active)
        {
            double r = sdf[v] - g.sdf0[v];
            if (r == 0.0) r = 0.0000001;
            acc[1] = r * r;
        }
        if (rv.use_ea)
        {
#pragma unroll
            for (int d = 0; d < 3; ++d)
            {
                const float wp = rv.ea_w[static_cast<int64_t>(d) * g.n + v];
                if (wp != 0.0f) { const double r = alb[v] - alb[g.nbr[static_cast<int64_t>(2 * d) * g.n + v]]; acc[2] += static_cast<double>(wp) * r * r; }
            }
        }
    }
    grid_reduce<3>(acc, site);
}


// ----------------------------------------------------------------------------------------------
// device-resident control of one GN iteration (round 2): the per-type weight normalisation, the LM bookkeeping of
// TrustRegionMinimizer (step validity, relative decrease, radius update, termination tests) and the result struct live on
// the device; the host enqueues a whole trial (PCG + model change + candidate cost + decision) and reads ONE struct back.
// ----------------------------------------------------------------------------------------------
enum { LM_RUNNING = 0, LM_ACCEPTED = 1, LM_TERMINATED = 2 };
struct IterDev
{
    I3DIterInfo info;
    double radius, decrease_factor, x_norm, g_norm;
    int invalid_steps;
    int state;            // LM_*
    int pcg_unfinished;   // k_lm_decide found the PCG still running: the host enqueues more iterations and decides again
    int precond_fail;     // a camera block of the block-Jacobi preconditioner was not SPD
};

// NLSSolver::normalizeCostTermWeights (nls_solver.cpp:379-394) + the cost at the initial point, from the (allreduced) row sums.
//   build_out: [0] sum raw E_g weights [1] sum raw w r^2 [2] valid E_g rows [3] active voxels
//   reg_out  : [0] n_Er [1] sum r_Er^2 [2] n_Es [3] sum r_Es^2 [4] n_Ea [5] sum w_Ea [6] sum w_Ea r^2 [7] n_free_sdf [8] n_free_alb
__global__ void k_type_weights(IterDev* __restrict__ it, const double* __restrict__ build_out, const double* __restrict__ reg_out, I3DParams P,
                               int64_t num_voxels, double* __restrict__ type_w)
{
    pdl_prologue();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    I3DIterInfo& info = it->info;
    memset(&info, 0, sizeof(info));
    it->precond_fail = 0;
    info.num_voxels = num_voxels;
    info.num_active = static_cast<int64_t>(build_out[3]);
    const double sums[4] = {build_out[0], reg_out[0], reg_out[2], reg_out[5]};
    const double raw_cost[4] = {build_out[1], reg_out[1], reg_out[3], reg_out[6]};
    info.type_residuals[0] = static_cast<int64_t>(build_out[2]); info.type_residuals[1] = static_cast<int64_t>(reg_out[0]);
    info.type_residuals[2] = static_cast<int64_t>(reg_out[2]); info.type_residuals[3] = static_cast<int64_t>(reg_out[4]);
    info.num_free_sdf = static_cast<int64_t>(reg_out[7]); info.num_free_albedo = static_cast<int64_t>(reg_out[8]);
    double cost0 = 0.0;
    for (int t = 0; t < 4; ++t)
    {
        const double tw = (sums[t] != 0.0) ? (P.lambda[t] / sums[t]) * 1000.0 : 0.0;
        type_w[t] = tw;
        info.type_sum_weights[t] = sums[t]; info.type_weights[t] = tw;
        info.type_costs[t] = 0.5 * tw * raw_cost[t];
        cost0 += info.type_costs[t];
    }
    info.cost_initial = cost0; info.cost_final = cost0;
    it->radius = P.initial_trust_region_radius; it->decrease_factor = 2.0; it->invalid_steps = 0; it->pcg_unfinished = 0;
    info.trust_region_radius = it->radius;
    info.termination = 2; info.lm_iterations = 0; info.step_accepted = 0; info.cg_iterations_total = 0;
    it->state = LM_RUNNING;
    if (info.num_active == 0) { it->state = LM_TERMINATED; info.termination = 4; }
}

// finish_out: [0] free parameters with a non-zero column [1] ||x||^2 over those [2] ||gradient||^2 (free unknowns)
__global__ void k_iter_finish(IterDev* __restrict__ it, const double* __restrict__ finish_out, I3DParams P)
{
    pdl_prologue();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    it->info.num_parameters = static_cast<int64_t>(finish_out[0]);
    it->x_norm = sqrt(finish_out[1]);
    it->g_norm = sqrt(finish_out[2]);
    if (it->state != LM_RUNNING) return;
    if (P.build_only) { it->state = LM_TERMINATED; it->info.termination = 4; }
    else if (it->g_norm <= P.gradient_tolerance) { it->state = LM_TERMINATED; it->info.termination = 1; }
}

// start of one LM trial: resets the PCG control block with the current radius (or halts everything if the loop is over)
__global__ void k_lm_begin(IterDev* __restrict__ it, CgCtl* __restrict__ ctl, int* __restrict__ fail_flag, I3DParams P)
{
    pdl_prologue();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    CgCtl c;
    memset(&c, 0, sizeof(c));
    if (it->state != LM_RUNNING) { c.done = 1; c.halt = 1; c.inv_radius = 1.0; *ctl = c; return; }
    it->info.lm_iterations += 1;
    it->pcg_unfinished = 0;
    c.inv_radius = 1.0 / it->radius; c.eta = P.eta;
    c.forced_iterations = P.forced_cg_iterations; c.max_iterations = P.max_linear_solver_iterations; c.min_iterations = P.min_linear_solver_iterations;
    *ctl = c;
    *fail_flag = 0;
}

// end of one LM trial (TrustRegionMinimizer's iteration body after the linear solve; see oracle.cpp "LM loop"):
//   cand: [0] ||delta||^2   eg_cost: [0] sum raw_w r^2   reg_cost: [0] E_r [1] E_s [2] E_a (raw)
__global__ void k_lm_decide(IterDev* __restrict__ it, const CgCtl* __restrict__ ctl, const int* __restrict__ fail_flag,
                            const double* __restrict__ cand_out, const double* __restrict__ eg_cost, const double* __restrict__ reg_cost,
                            const double* __restrict__ type_w, I3DParams P)
{
    pdl_prologue();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (it->state != LM_RUNNING) return;
    I3DIterInfo& info = it->info;
    const int precond_fail = *fail_flag;
    const int max_it = P.forced_cg_iterations > 0 ? P.forced_cg_iterations : P.max_linear_solver_iterations;
    if (!ctl->done && !precond_fail && ctl->it < max_it) { it->pcg_unfinished = 1; return; }
    it->pcg_unfinished = 0;
    const int slot = min(info.lm_iterations - 1, I3D_MAX_LM_STEPS - 1);
    info.cg_iterations[slot] = ctl->it; info.cg_iterations_total += ctl->it;
    if (precond_fail) { info.termination = 3; it->state = LM_TERMINATED; it->precond_fail = 1; return; }
    bool step_valid = (ctl->status != 1);
    double model_cost_change = 0.0, cand = 0.0, step_norm = 0.0;
    if (step_valid)
    {
        // model cost change -(J'd).(f + J'd/2) for d = -x, from the scalars the PCG maintains instead of another pass over the
        // Jacobian:  x.b - x.(J'^T J' x)/2  with  J'^T J' x = (b - r) - D^2 x   =>   (x.(b + r) + x.D^2 x) / 2,  and Q1 = -x.(b + r)
        // (r = b - A x is the recursively updated PCG residual, refreshed exactly every residual_reset_period iterations)
        model_cost_change = 0.5 * (ctl->xd2x - ctl->Q1);
        cand = 0.5 * (type_w[0] * eg_cost[0] + type_w[1] * reg_cost[0] + type_w[2] * reg_cost[1] + type_w[3] * reg_cost[2]);
        step_norm = sqrt(cand_out[0]);
        if (!isfinite(step_norm)) step_valid = false;
        else step_valid = model_cost_change > 0.0;
    }
    info.model_cost_change[slot] = model_cost_change;
    const bool last_trial = info.lm_iterations >= P.lm_steps;
    if (!step_valid)
    {
        if (++it->invalid_steps >= P.max_consecutive_invalid_steps) { info.termination = 3; it->state = LM_TERMINATED; return; }
        it->radius *= 0.5; info.trust_region_radius = it->radius;
        if (it->radius <= P.min_trust_region_radius) { info.termination = 1; it->state = LM_TERMINATED; return; }
        if (last_trial) it->state = LM_TERMINATED;
        return;
    }
    it->invalid_steps = 0;
    info.candidate_cost[slot] = cand; info.step_norm = step_norm;
    if (step_norm <= P.parameter_tolerance * (it->x_norm + P.parameter_tolerance)) { info.termination = 1; it->state = LM_TERMINATED; return; }
    const double cost0 = info.cost_initial;
    const double cost_change = cost0 - cand;
    if (fabs(cost_change) <= P.function_tolerance * cost0) { info.termination = 1; it->state = LM_TERMINATED; return; }
    const double rho_q = cost_change / model_cost_change;
    info.relative_decrease[slot] = rho_q;
    if (rho_q > P.min_relative_decrease)
    {
        const double t = 2.0 * rho_q - 1.0;
        double radius = it->radius / fmax(1.0 / 3.0, 1.0 - t * t * t);
        radius = fmin(P.max_trust_region_radius, radius);
        it->radius = radius;
        info.trust_region_radius = radius; info.cost_final = cand; info.step_accepted = 1; info.termination = 0;
        it->state = LM_ACCEPTED;
        return;
    }
    it->radius = it->radius / it->decrease_factor; it->decrease_factor *= 2.0; info.trust_region_radius = it->radius;
    if (it->radius <= P.min_trust_region_radius) { info.termination = 1; it->state = LM_TERMINATED; return; }
    if (last_trial) it->state = LM_TERMINATED;
}

} // namespace i3d
