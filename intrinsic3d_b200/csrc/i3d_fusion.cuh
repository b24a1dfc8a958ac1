/*
 * i3d_fusion.cuh — RGB-D fusion into the voxel grid on the device (DESIGN.md §6h).
 *
 * Restates the chain AppFusion::fuseSDF runs per frame (apps/src/app_fusion.cpp:107-200, paths below relative to libintrinsic3d/):
 *   k_fuse_erode      erodeDiscontinuities(depth, window, 0.5)          src/rgbd/processing.cpp:184-235
 *   k_fuse_normals    computeNormals(K, depth, 0.3) (vertex map on the fly)  :49-126
 *   k_fuse_alloc      SparseVoxelGrid::alloc (ray march, 3x3x3 blocks)   src/sparse_voxel_grid.cpp:398-467
 *   k_fuse_integrate  SparseVoxelGrid::integrate's per-voxel update      :300-395
 * and, after all frames,
 *   k_fuse_correct    SDFAlgorithms::correctSDF as Jacobi sweeps        src/sdf/algorithms.cpp:260-337
 *   k_fuse_sort_keys / k_fuse_convert   clearInvalidVoxels (:342-363) + SDFAlgorithms::convert, in canonical order
 *
 * Float arithmetic is written operation by operation with FM/FA/FS/FD (no contraction) so that it rounds like the float CPU
 * restatement in tests/native/fusion_oracle.cpp; vector sums run left to right, as everywhere in this engine.
 *
 * The in-progress volume is a Voxel {float sdf, float weight, uchar3 colour} per allocated voxel, indexed in the (nondeterministic)
 * order in which hash slots were claimed.  Nothing downstream depends on that order: the per-voxel update reads only the voxel itself,
 * the Jacobi sweep reads only the previous sweep, and every output is gathered in canonical 8^3-brick-major order
 * (sort key fuse_order_key).
 */
#pragma once
#include "i3d_fusion_view.cuh"

namespace i3d
{

constexpr int kFuseMaxProbe = 128;            // a longer linear probe means the table is too full: grow it
constexpr int kFuseCoordLimit = (1 << 20) - 2; // centre voxels beyond this would put a block neighbour outside pack_key's range

// what SparseVoxelGrid::integrate and alloc read per frame
struct FuseCam { int W, H; float fx, fy, cx, cy; };
struct FuseFrame
{
    float R_cw[9], t_cw[3];       // camera -> world (alloc)
    float R_wc[9], t_wc[3];       // world -> camera (integrate), supplied by the caller
    int bounds[6];                // computeFrustumBounds, inclusive voxel bounds x0,x1,y0,y1,z0,z1
};
struct FuseConst
{
    float voxel_size, inv_voxel_size, truncation, ray_step;
    float depth_min, depth_max, weight_sample;
    float clip[6];
    int use_clip;
};
struct FuseTable
{
    unsigned long long* keys; unsigned* vals; uint64_t mask;
    int* count;                    // allocated voxels
    int* status;                   // bit 0: overflow (grow and re-run), bit 1: coordinate outside the packable range
    int limit;                     // count at which the table counts as full
};
struct FuseVolume
{
    int32_t* x; int32_t* y; int32_t* z;
    float* sdf; float* weight; uchar4* rgb;
};

// saturating float -> int toward zero: the (int) cast of nv::round / the reference's casts for every value that fits
__device__ __forceinline__ int fuse_f2i(float v) { return __float2int_rz(v); }

// SparseVoxelGrid::worldToVoxel (sparse_voxel_grid.cpp:211-220) = nv::round(p * (1 / voxel_size)) (include/nv/mat.h:90):
// (v + 0.5f).cast<int>() truncates toward zero, so (-1, -0.5] maps to 0
__device__ __forceinline__ int fuse_w2v(float p, float inv_vs) { return fuse_f2i(FA(FM(p, inv_vs), 0.5f)); }

__device__ __forceinline__ bool fuse_in_bounds(const int b[6], int x, int y, int z)
{
    return !(x < b[0] || x > b[1] || y < b[2] || y > b[3] || z < b[4] || z > b[5]);
}

__device__ __forceinline__ void fuse_xform(const float R[9], const float t[3], const float p[3], float q[3])
{
#pragma unroll
    for (int k = 0; k < 3; ++k) q[k] = FA(FA(FA(FM(R[3 * k], p[0]), FM(R[3 * k + 1], p[1])), FM(R[3 * k + 2], p[2])), t[k]);
}

// 64-bit canonical order key: (bz, by, bx, lz, ly, lx) with b = floor(c / 8), l = c - 8 b; c + 2^20 >= 0 for every packable c
__host__ __device__ __forceinline__ unsigned long long fuse_order_key(int x, int y, int z)
{
    const unsigned long long ux = static_cast<unsigned long long>(x + (1 << 20)), uy = static_cast<unsigned long long>(y + (1 << 20)),
                             uz = static_cast<unsigned long long>(z + (1 << 20));
    return ((uz >> 3) << 46) | ((uy >> 3) << 28) | ((ux >> 3) << 10) | ((uz & 7ull) << 6) | ((uy & 7ull) << 3) | (ux & 7ull);
}

// ---- erodeDiscontinuities (processing.cpp:184-235): a pixel survives iff every pixel of its clipped window is non-zero and within 0.5 m
__global__ void k_fuse_erode(int W, int H, int window, const float* __restrict__ din, float* __restrict__ dout)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= static_cast<int64_t>(W) * H) return;
    const int y = static_cast<int>(i / W), x = static_cast<int>(i - static_cast<int64_t>(y) * W);
    const float d_ref = din[i];
    bool valid = d_ref != 0.0f;
    if (valid && window > 0)
        for (int v = max(0, y - window); v <= min(y + window, H - 1) && valid; ++v)
            for (int u = max(0, x - window); u <= min(x + window, W - 1); ++u)
            {
                const float d = din[static_cast<int64_t>(v) * W + u];
                if (d == 0.0f || fabsf(FS(d, d_ref)) > 0.5f) { valid = false; break; }
            }
    dout[i] = valid ? d_ref : 0.0f;
}

// computeNormals(K, depth, 0.3) (processing.cpp:49-126) by depth_normal
__global__ void k_fuse_normals(FuseCam cam, const float* __restrict__ depth, float* __restrict__ nrm /* [H][W][3] */)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= static_cast<int64_t>(cam.W) * cam.H) return;
    const float3 n = depth_normal(depth, cam.W, cam.H, cam.fx, cam.fy, cam.cx, cam.cy, i);
    nrm[3 * i] = n.x; nrm[3 * i + 1] = n.y; nrm[3 * i + 2] = n.z;
}

// insert-or-find; returns the slot, or -1 after raising the overflow status
__device__ __forceinline__ int64_t fuse_insert(const FuseTable& t, const FuseVolume& vol, int x, int y, int z)
{
    const unsigned long long key = pack_key(x, y, z);
    uint64_t slot = mix64(key) & t.mask;
    for (int probe = 0; probe < kFuseMaxProbe; ++probe)
    {
        unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(&t.keys[slot]);
        if (k == kEmptyKey)
        {
            k = atomicCAS(&t.keys[slot], kEmptyKey, key);
            if (k == kEmptyKey)
            {
                const int idx = atomicAdd(t.count, 1);           // the volume arrays hold one entry per slot: idx < capacity always
                atomicOr(&t.vals[slot], static_cast<unsigned>(idx));
                vol.x[idx] = x; vol.y[idx] = y; vol.z[idx] = z;
                vol.sdf[idx] = 0.0f; vol.weight[idx] = 0.0f; vol.rgb[idx] = make_uchar4(0, 0, 0, 0);   // Voxel() (sparse_voxel_grid.h:56-62)
                if (idx + 1 >= t.limit) atomicOr(t.status, 1);
                return static_cast<int64_t>(slot);
            }
        }
        if (k == key) return static_cast<int64_t>(slot);
        slot = (slot + 1) & t.mask;
    }
    atomicOr(t.status, 1);
    return -1;
}

// SparseVoxelGrid::alloc (sparse_voxel_grid.cpp:398-467), one thread per pixel.  use_block_bit: a centre whose block is already complete
// inserts nothing (the voxel set is the same: the block exists); it is off on the re-run after a growth, where an aborted thread may
// have left a block incomplete without setting the bit — bits are only set after all 27 inserts, so this is belt and braces.
__global__ void k_fuse_alloc(FuseCam cam, FuseFrame fr, FuseConst c, const float* __restrict__ depth, FuseTable t,
                             FuseVolume vol, int use_block_bit)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= static_cast<int64_t>(cam.W) * cam.H) return;
    const float d = depth[i];
    if (d == 0.0f) return;
    const int y = static_cast<int>(i / cam.W), x = static_cast<int>(i - static_cast<int64_t>(y) * cam.W);
    // Camera::unproject2(x, y, 1.0f) (src/camera.cpp:191-199)
    const float pc[3] = {FD(FS(static_cast<float>(x), cam.cx), cam.fx), FD(FS(static_cast<float>(y), cam.cy), cam.fy), 1.0f};
    int last[3] = {0, 0, 0};                              // pos_grid_last = Vec3i::Zero(): a first sample in voxel (0,0,0) is skipped
    for (float d_off = -c.truncation; d_off <= c.truncation; d_off = FA(d_off, c.ray_step))
    {
        if (*reinterpret_cast<volatile int*>(t.status)) return;
        const float s = FA(d, d_off);
        const float pr[3] = {FM(pc[0], s), FM(pc[1], s), FM(pc[2], s)};
        float pw[3];
        fuse_xform(fr.R_cw, fr.t_cw, pr, pw);
        const int g[3] = {fuse_w2v(pw[0], c.inv_voxel_size), fuse_w2v(pw[1], c.inv_voxel_size), fuse_w2v(pw[2], c.inv_voxel_size)};
        if (g[0] == last[0] && g[1] == last[1] && g[2] == last[2]) continue;
        last[0] = g[0]; last[1] = g[1]; last[2] = g[2];
        if (!fuse_in_bounds(fr.bounds, g[0], g[1], g[2])) continue;
        if (c.use_clip)
        {
            const float w0 = FM(static_cast<float>(g[0]), c.voxel_size), w1 = FM(static_cast<float>(g[1]), c.voxel_size), w2 = FM(static_cast<float>(g[2]), c.voxel_size);
            if (w0 < c.clip[0] || w0 > c.clip[1] || w1 < c.clip[2] || w1 > c.clip[3] || w2 < c.clip[4] || w2 > c.clip[5]) continue;
        }
        if (abs(g[0]) > kFuseCoordLimit || abs(g[1]) > kFuseCoordLimit || abs(g[2]) > kFuseCoordLimit) { atomicOr(t.status, 2); return; }
        const int64_t sc = fuse_insert(t, vol, g[0], g[1], g[2]);
        if (sc < 0) return;
        if (use_block_bit && (*reinterpret_cast<volatile unsigned*>(&t.vals[sc]) & kFuseBlockBit)) continue;
        for (int dz = -1; dz <= 1; ++dz)
            for (int dy = -1; dy <= 1; ++dy)
                for (int dx = -1; dx <= 1; ++dx)
                {
                    if (dx == 0 && dy == 0 && dz == 0) continue;
                    if (fuse_insert(t, vol, g[0] + dx, g[1] + dy, g[2] + dz) < 0) return;
                }
        atomicOr(&t.vals[sc], kFuseBlockBit);
    }
}

// math::robustKernel(val, 2) (src/math.cpp:43-47)
__device__ __forceinline__ float fuse_robust(float v)
{
    const float div = FA(1.0f, FM(2.0f, v));
    return FD(1.0f, FM(FM(div, div), div));
}

// SparseVoxelGrid::integrate's per-voxel body (sparse_voxel_grid.cpp:316-392), one thread per allocated voxel.
// normals may be NULL (weight_sample == 0: never read).  bgr: interleaved B,G,R of the colour camera.
__global__ void __launch_bounds__(kThreads) k_fuse_integrate(int64_t n, FuseCam dcam, FuseCam ccam, FuseFrame fr, FuseConst c,
                                                             const float* __restrict__ depth, const float* __restrict__ normals,
                                                             const uint8_t* __restrict__ bgr, FuseVolume vol)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    const int X = vol.x[i], Y = vol.y[i], Z = vol.z[i];
    if (!fuse_in_bounds(fr.bounds, X, Y, Z)) return;
    const float pw[3] = {FM(static_cast<float>(X), c.voxel_size), FM(static_cast<float>(Y), c.voxel_size), FM(static_cast<float>(Z), c.voxel_size)};
    float p[3];
    fuse_xform(fr.R_wc, fr.t_wc, pw, p);
    if (p[2] < 0.0f) return;
    // round(depth_cam.project2(p)) (src/camera.cpp:157-162)
    const int u = fuse_f2i(FA(FA(FD(FM(p[0], dcam.fx), p[2]), dcam.cx), 0.5f));
    const int v = fuse_f2i(FA(FA(FD(FM(p[1], dcam.fy), p[2]), dcam.cy), 0.5f));
    if (u < 0 || v < 0 || u >= dcam.W || v >= dcam.H) return;
    const int64_t pix = static_cast<int64_t>(v) * dcam.W + u;
    const float d = depth[pix];
    if (d <= 0.0f) return;
    const float sdf = FS(d, p[2]);
    if (sdf <= -c.truncation) return;
    const float tsdf = sdf >= 0.0f ? fminf(c.truncation, sdf) : fmaxf(-c.truncation, sdf);
    float wu = 1.0f;
    if (c.weight_sample > 0.0f)
    {
        const float nx = normals[3 * pix], ny = normals[3 * pix + 1], nz = normals[3 * pix + 2];
        float q[3] = {p[0], p[1], p[2]};
        const float sq = FA(FA(FM(q[0], q[0]), FM(q[1], q[1])), FM(q[2], q[2]));
        if (sq > 0.0f) { const float l = __fsqrt_rn(sq); q[0] = FD(q[0], l); q[1] = FD(q[1], l); q[2] = FD(q[2], l); }
        float w_normal = FS(1.0f, fabsf(FA(FA(FM(q[0], nx), FM(q[1], ny)), FM(q[2], nz))));
        w_normal = fmaxf(fminf(w_normal, 1.0f), 0.0f);
        w_normal = fmaxf(FM(c.weight_sample, fuse_robust(w_normal)), 1.0f);
        const float w_dist = fmaxf(FM(c.weight_sample, fuse_robust(FD(FM(2.0f, fabsf(tsdf)), c.truncation))), 1.0f);
        const float d_norm = FD(FS(d, c.depth_min), FS(c.depth_max, c.depth_min));
        const float w_depth = fmaxf(FM(c.weight_sample, FS(1.0f, d_norm)), 1.0f);
        wu = fmaxf(FD(FA(FA(w_normal, w_dist), w_depth), 3.0f), 3.0f);
    }
    const float w_old = vol.weight[i];
    const float w_new = FA(w_old, wu);
    vol.sdf[i] = FD(FA(FM(vol.sdf[i], w_old), FM(sdf, wu)), w_new);      // running mean of the unclamped sdf
    const int cu = fuse_f2i(FA(FA(FD(FM(p[0], ccam.fx), p[2]), ccam.cx), 0.5f));
    const int cv = fuse_f2i(FA(FA(FD(FM(p[1], ccam.fy), p[2]), ccam.cy), 0.5f));
    if (cu >= 0 && cv >= 0 && cu < ccam.W && cv < ccam.H)
    {
        const uint8_t* px = bgr + (static_cast<int64_t>(cv) * ccam.W + cu) * 3;
        uchar4 o = vol.rgb[i];
        const float cn[3] = {static_cast<float>(px[2]), static_cast<float>(px[1]), static_cast<float>(px[0])};
        const float r = FD(FA(FM(static_cast<float>(o.x), w_old), FM(cn[0], wu)), w_new);
        const float g = FD(FA(FM(static_cast<float>(o.y), w_old), FM(cn[1], wu)), w_new);
        const float b = FD(FA(FM(static_cast<float>(o.z), w_old), FM(cn[2], wu)), w_new);
        o.x = static_cast<unsigned char>(fuse_f2i(r)); o.y = static_cast<unsigned char>(fuse_f2i(g)); o.z = static_cast<unsigned char>(fuse_f2i(b));
        vol.rgb[i] = o;
    }
    vol.weight[i] = w_new;
}

// fusion table after a growth: re-insert every claimed slot (key and value, block bit included) into the new table
__global__ void k_fuse_rehash(uint64_t old_cap, const unsigned long long* __restrict__ okeys, const unsigned* __restrict__ ovals,
                              unsigned long long* __restrict__ keys, unsigned* __restrict__ vals, uint64_t mask)
{
    const int64_t s = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (s >= static_cast<int64_t>(old_cap)) return;
    const unsigned long long key = okeys[s];
    if (key == kEmptyKey) return;
    uint64_t slot = mix64(key) & mask;
    while (atomicCAS(&keys[slot], kEmptyKey, key) != kEmptyKey) slot = (slot + 1) & mask;
    vals[slot] = ovals[s];
}

// One Jacobi sweep of SDFAlgorithms::correctSDF (algorithms.cpp:260-337): every valid voxel compares its 26 neighbours in (k, j, i)
// order against its sweep-start value; the LAST qualifying neighbour wins (weight := 1).  Neighbours are read from the previous sweep.
// The reference's weight == 0 / isinf branch cannot run (valid() requires weight > 0) and is not restated.  *changed: any update.
__global__ void k_fuse_correct(int64_t n, float vs, const unsigned long long* __restrict__ keys, const unsigned* __restrict__ vals,
                               uint64_t mask, const int32_t* __restrict__ X, const int32_t* __restrict__ Y, const int32_t* __restrict__ Z,
                               const float* __restrict__ sdf_in, const float* __restrict__ w_in,
                               float* __restrict__ sdf_out, float* __restrict__ w_out, int* __restrict__ changed)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    const float w0 = w_in[i];
    float s_new = sdf_in[i], w_new = w0;
    if (w0 > 0.0f)
    {
        const int x = X[i], y = Y[i], z = Z[i];
        const double sdf = static_cast<double>(sdf_in[i]);
        const double sgn = sdf >= 0.0 ? 1.0 : -1.0;
        const float cx = FM(static_cast<float>(x), vs), cy = FM(static_cast<float>(y), vs), cz = FM(static_cast<float>(z), vs);
        bool upd = false;
        double best = 0.0;
        for (int k = -1; k <= 1; ++k)
            for (int j = -1; j <= 1; ++j)
                for (int ii = -1; ii <= 1; ++ii)
                {
                    if (k == 0 && j == 0 && ii == 0) continue;
                    const int32_t nb = fuse_find(keys, vals, mask, x + ii, y + j, z + k);
                    if (nb < 0 || !(w_in[nb] > 0.0f)) continue;
                    const double sdf_nb = static_cast<double>(sdf_in[nb]);
                    const double sgn_nb = sdf_nb >= 0.0 ? 1.0 : -1.0;
                    const float dx = FS(cx, FM(static_cast<float>(x + ii), vs)), dy = FS(cy, FM(static_cast<float>(y + j), vs)),
                                dz = FS(cz, FM(static_cast<float>(z + k), vs));
                    const float len = __fsqrt_rn(FA(FA(FM(dx, dx), FM(dy, dy)), FM(dz, dz)));
                    const double dist_nb = __dadd_rn(sdf_nb, __dmul_rn(sgn_nb, static_cast<double>(len)));
                    if (fabs(dist_nb) < fabs(sdf) && sgn == sgn_nb) { best = dist_nb; upd = true; }
                }
        if (upd) { s_new = static_cast<float>(best); w_new = 1.0f; *changed = 1; }
    }
    sdf_out[i] = s_new; w_out[i] = w_new;
}

// canonical order keys; `valid_only`: voxels with weight <= 0 (clearInvalidVoxels) get the largest key so they sort last
__global__ void k_fuse_sort_keys(int64_t n, const int32_t* __restrict__ X, const int32_t* __restrict__ Y, const int32_t* __restrict__ Z,
                                 const float* __restrict__ w, int valid_only, unsigned long long* __restrict__ keys, int32_t* __restrict__ idx,
                                 int* __restrict__ num_valid)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    const bool keep = !valid_only || w[i] > 0.0f;
    keys[i] = keep ? fuse_order_key(X[i], Y[i], Z[i]) : ~0ull;
    idx[i] = static_cast<int32_t>(i);
    if (keep && valid_only)
    {
        const unsigned m = __ballot_sync(__activemask(), true);
        if ((threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(num_valid, __popc(m));
    }
}

// SDFAlgorithms::convert (Voxel -> VoxelSBR, as intrinsic3d_b200/host/algorithms.cpp:79-93): sdf0 = sdf_refined = (double) sdf,
// albedo 0.6, weight, colour; voxel i of the result is volume entry order[i]
__global__ void k_fuse_convert(int64_t m, const int32_t* __restrict__ order, FuseVolume vol, VoxelArrays out)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= m) return;
    const int32_t v = order[i];
    out.x[i] = vol.x[v]; out.y[i] = vol.y[v]; out.z[i] = vol.z[v];
    const double s = static_cast<double>(vol.sdf[v]);
    out.sdf0[i] = s; out.sdf[i] = s; out.albedo[i] = 0.6;
    out.weight[i] = vol.weight[v]; out.rgb[i] = vol.rgb[v];
}

// the in-progress volume in canonical order, interleaved for the host (i3d_debug_get_fusion_volume)
__global__ void k_fuse_gather(int64_t m, const int32_t* __restrict__ order, FuseVolume vol, int32_t* __restrict__ xyz, float* __restrict__ sdf,
                              float* __restrict__ w, uint8_t* __restrict__ rgb3)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= m) return;
    const int32_t v = order[i];
    xyz[3 * i] = vol.x[v]; xyz[3 * i + 1] = vol.y[v]; xyz[3 * i + 2] = vol.z[v];
    sdf[i] = vol.sdf[v]; w[i] = vol.weight[v];
    const uchar4 c = vol.rgb[v];
    rgb3[3 * i] = c.x; rgb3[3 * i + 1] = c.y; rgb3[3 * i + 2] = c.z;
}

} // namespace i3d
