/*
 * i3d_fusion.cu — the RGB-D fusion: its kernels (i3d_fusion.cuh), the canonical sort and the host code that sequences them (i3d_fusion.h).
 * The layout of the fusion's hash table (slot values, the control block, the load factor and the growth) is known only here and in
 * i3d_fusion.cuh.
 */
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>

#include "i3d_fusion.cuh"
#include "i3d_fusion.h"

#include <cub/device/device_radix_sort.cuh>

namespace i3d
{
namespace
{
FuseTable fuse_table(const FusionState& fs)
{
    FuseTable t;
    t.keys = fs.keys.p; t.vals = fs.vals.p; t.mask = fs.cap - 1; t.count = fs.ctl.p; t.status = fs.ctl.p + 1;
    t.limit = static_cast<int>(fs.cap / 2);              // load factor 0.5
    return t;
}
FuseVolume fuse_volume(const FusionState& fs) { return FuseVolume{fs.x.p, fs.y.p, fs.z.p, fs.sdf.p, fs.w.p, fs.rgb.p}; }

FuseConst fuse_const(const I3DFusionParams& P)
{
    FuseConst c;
    c.voxel_size = P.voxel_size; c.inv_voxel_size = 1.0f / P.voxel_size;
    c.truncation = P.voxel_size * 5.0f; c.ray_step = P.voxel_size * 0.25f;      // sparse_voxel_grid.cpp:48, :403
    c.depth_min = P.depth_min; c.depth_max = P.depth_max; c.weight_sample = P.integration_weight_sample;
    float sq = 0.0f;
    for (int k = 0; k < 6; ++k) { c.clip[k] = P.clip_bounds[k]; sq += P.clip_bounds[k] * P.clip_bounds[k]; }
    c.use_clip = sq > 0.0f ? 1 : 0;                      // clip_bounds.norm() > 0 (app_fusion.cpp:138)
    return c;
}

// (int) cast of a float, saturating where the C++ cast is undefined (same values as __float2int_rz on the device)
int fuse_f2i_host(float v)
{
    if (!(v == v)) return 0;
    if (v >= 2147483648.0f) return INT_MAX;
    if (v < -2147483648.0f) return INT_MIN;
    return static_cast<int>(v);
}

// SparseVoxelGrid::computeFrustumBounds (sparse_voxel_grid.cpp:572-602) with math::computeFrustumPoints (src/math.cpp:131-148).
// floor / ceil act on the WORLD point in metres before worldToVoxel, so the bounds are whole-metre aligned.
void fuse_frustum_bounds(const I3DFusionCamera& cam, float dmin, float dmax, float vs, const float R[9], const float t[3], int b[6])
{
    const float inv = 1.0f / vs;
    const int px[4] = {0, cam.width - 1, cam.width - 1, 0}, py[4] = {0, 0, cam.height - 1, cam.height - 1};
    b[0] = b[2] = b[4] = INT_MAX; b[1] = b[3] = b[5] = INT_MIN;
    for (int i = 0; i < 8; ++i)
    {
        const float d = i < 4 ? dmin : dmax;
        float c[3] = {0.0f, 0.0f, 0.0f};
        if (d != 0.0f)                                   // Camera::unproject2 returns zero for depth 0
        {
            const float x = (static_cast<float>(px[i & 3]) - cam.cx) / cam.fx, y = (static_cast<float>(py[i & 3]) - cam.cy) / cam.fy;
            c[0] = d * x; c[1] = d * y; c[2] = d;
        }
        for (int k = 0; k < 3; ++k)
        {
            float p = R[3 * k] * c[0];
            p = p + R[3 * k + 1] * c[1];
            p = p + R[3 * k + 2] * c[2];
            p = p + t[k];
            const int pl = fuse_f2i_host(static_cast<float>(fuse_f2i_host(std::floor(p))) * inv + 0.5f);
            const int pu = fuse_f2i_host(static_cast<float>(fuse_f2i_host(std::ceil(p))) * inv + 0.5f);
            b[2 * k] = std::min(b[2 * k], std::min(pl, pu));
            b[2 * k + 1] = std::max(b[2 * k + 1], std::max(pl, pu));
        }
    }
}

void fuse_reset_table(FusionState& fs, uint64_t cap, cudaStream_t st)
{
    fs.keys.ensure(cap); fs.vals.ensure(cap); fs.ctl.ensure(4);
    fs.x.ensure(cap); fs.y.ensure(cap); fs.z.ensure(cap); fs.sdf.ensure(cap); fs.w.ensure(cap); fs.rgb.ensure(cap);
    fs.cap = cap;
    CK(cudaMemsetAsync(fs.keys.p, 0xFF, cap * sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(fs.vals.p, 0, cap * sizeof(unsigned), st));
    CK(cudaMemsetAsync(fs.ctl.p, 0, 4 * sizeof(int), st));
    CK(cudaStreamSynchronize(st));
}

template <class T>
void fuse_grow_copy(Dev<T>& a, size_t cap, size_t keep, cudaStream_t st)
{
    Dev<T> b;
    b.ensure(cap);
    if (keep) CK(cudaMemcpyAsync(b.p, a.p, keep * sizeof(T), cudaMemcpyDeviceToDevice, st));
    CK(cudaStreamSynchronize(st));
    a.swap(b);
}

// new table of `cap` slots: every claimed slot (key, voxel index, block bit) is re-inserted; the volume keeps its indices
void fuse_grow_table(FusionState& fs, uint64_t cap, cudaStream_t st)
{
    const size_t keep = static_cast<size_t>(fs.n);
    Dev<unsigned long long> nk; Dev<unsigned> nv;
    nk.ensure(cap); nv.ensure(cap);
    CK(cudaMemsetAsync(nk.p, 0xFF, cap * sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(nv.p, 0, cap * sizeof(unsigned), st));
    k_fuse_rehash<<<blocks_for(fs.cap), kThreads, 0, st>>>(fs.cap, fs.keys.p, fs.vals.p, nk.p, nv.p, cap - 1);
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    fs.keys.swap(nk); fs.vals.swap(nv);
    fuse_grow_copy(fs.x, cap, keep, st); fuse_grow_copy(fs.y, cap, keep, st); fuse_grow_copy(fs.z, cap, keep, st);
    fuse_grow_copy(fs.sdf, cap, keep, st); fuse_grow_copy(fs.w, cap, keep, st); fuse_grow_copy(fs.rgb, cap, keep, st);
    fs.cap = cap;
}
} // namespace

void fusion::begin(FusionState& fs, Timing& tm, const I3DFusionParams& P, cudaStream_t st)
{
    fs.p = P;
    uint64_t cap = P.initial_capacity > 0 ? 64 : (1ull << 22);
    while (cap < static_cast<uint64_t>(P.initial_capacity)) cap <<= 1;
    fuse_reset_table(fs, cap, st);
    fs.n = 0;
    fs.motion = 0;
    fs.ref_id = -1;
    begin_timing(tm, {"fusion_prep", "fusion_alloc", "fusion_integrate", "fusion_correct", "fusion_finish", "fusion_growths", "fusion_sweeps"});
}

int fusion::integrate_host(FusionState& fs, Timing& tm, int F, const I3DFusionCamera& dc, const float* depth, const I3DFusionCamera& cc,
                           const uint8_t* bgr, const float* pose_cam_to_world, const float* pose_world_to_cam, std::string& error, cudaStream_t st)
{
    const size_t dimg = static_cast<size_t>(dc.width) * dc.height;
    const size_t cimg = static_cast<size_t>(cc.width) * cc.height * 3;
    fs.depth_in.ensure(dimg * F); fs.bgr.ensure(cimg * F);
    CK(cudaMemcpyAsync(fs.depth_in.p, depth, dimg * F * sizeof(float), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(fs.bgr.p, bgr, cimg * F, cudaMemcpyHostToDevice, st));
    return integrate(fs, tm, F, dc, fs.depth_in.p, cc, fs.bgr.p, nullptr, pose_cam_to_world, pose_world_to_cam, error, st);
}

int fusion::integrate(FusionState& fs, Timing& tm, int n, const I3DFusionCamera& depth_cam, const float* depth, const I3DFusionCamera& color_cam,
                      const uint8_t* bgr, const int32_t* ids, const float* pose_cam_to_world, const float* pose_world_to_cam, std::string& error,
                      cudaStream_t st)
{
    const I3DFusionParams& P = fs.p;
    const size_t dimg = static_cast<size_t>(depth_cam.width) * depth_cam.height;
    const size_t cimg = static_cast<size_t>(color_cam.width) * color_cam.height * 3;
    fs.depth.ensure(dimg);
    const bool want_normals = P.integration_weight_sample > 0.0f;
    if (want_normals) fs.nrm.ensure(3 * dimg);
    const FuseCam dc{depth_cam.width, depth_cam.height, depth_cam.fx, depth_cam.fy, depth_cam.cx, depth_cam.cy};
    const FuseCam cc{color_cam.width, color_cam.height, color_cam.fx, color_cam.fy, color_cam.cx, color_cam.cy};
    const FuseConst c = fuse_const(P);
    fs.motion = 0;
    fs.ref_id = -1;
    begin_timing(tm, {});                        // the fusion phases were reset by begin
    for (int f = 0; f < n; ++f)
    {
        const size_t src = static_cast<size_t>(ids ? ids[f] : f);
        FuseFrame fr;
        std::memcpy(fr.R_cw, pose_cam_to_world + 12 * f, 9 * sizeof(float)); std::memcpy(fr.t_cw, pose_cam_to_world + 12 * f + 9, 3 * sizeof(float));
        std::memcpy(fr.R_wc, pose_world_to_cam + 12 * f, 9 * sizeof(float)); std::memcpy(fr.t_wc, pose_world_to_cam + 12 * f + 9, 3 * sizeof(float));
        fuse_frustum_bounds(depth_cam, P.depth_min, P.depth_max, P.voxel_size, fr.R_cw, fr.t_cw, fr.bounds);
        {
            Timer t(tm, st, "fusion_prep");
            k_fuse_erode<<<blocks_for(dimg), kThreads, 0, st>>>(dc.W, dc.H, P.discont_window_size, depth + dimg * src, fs.depth.p);
            if (want_normals) k_fuse_normals<<<blocks_for(dimg), kThreads, 0, st>>>(dc, fs.depth.p, fs.nrm.p);
        }
        int ctl[2] = {0, 0};
        for (int attempt = 0;; ++attempt)
        {
            {
                Timer t(tm, st, "fusion_alloc");
                CK(cudaMemsetAsync(fs.ctl.p + 1, 0, sizeof(int), st));
                k_fuse_alloc<<<blocks_for(dimg), kThreads, 0, st>>>(dc, fr, c, fs.depth.p, fuse_table(fs), fuse_volume(fs), attempt == 0 ? 1 : 0);
                CK(cudaMemcpyAsync(ctl, fs.ctl.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
            }
            collect_kernel_times(tm, st);               // synchronises: ctl is on the host
            CK(cudaGetLastError());
            fs.n = ctl[0];
            if (ctl[1] & 2)
            {
                char buf[256];
                std::snprintf(buf, sizeof(buf), "frame %d allocates voxels outside the +-2^20 coordinate range of the device hash (voxel size %g); "
                              "the fusion is ended", f, static_cast<double>(P.voxel_size));
                error = buf;
                return 1;
            }
            if (!(ctl[1] & 1)) break;
            // the table is too full: grow it, then run this frame's allocation again (the voxel set is a union: re-inserting is harmless)
            uint64_t cap = fs.cap * 2;
            while (static_cast<uint64_t>(fs.n) * 4 > cap) cap <<= 1;
            if (cap > (1ull << 31)) { error = "more than 2^30 allocated voxels; the fusion is ended"; return 1; }
            fuse_grow_table(fs, cap, st);
            tm.phases["fusion_growths"].count += 1;
        }
        {
            Timer t(tm, st, "fusion_integrate");
            if (fs.n > 0)
                k_fuse_integrate<<<blocks_for(static_cast<size_t>(fs.n)), kThreads, 0, st>>>(fs.n, dc, cc, fr, c, fs.depth.p,
                                                                                            want_normals ? fs.nrm.p : nullptr, bgr + cimg * src,
                                                                                            fuse_volume(fs));
        }
    }
    collect_kernel_times(tm, st);
    CK(cudaGetLastError());
    return 0;
}

void fusion::correct(FusionState& fs, Timing& tm, cudaStream_t st)
{
    const int64_t n = fs.n;
    if (n <= 0) return;
    Timer t(tm, st, "fusion_correct");
    fs.sdf2.ensure(fs.sdf.cap); fs.w2.ensure(fs.w.cap);
    for (int it = 0; it < fs.p.correct_sdf_iterations; ++it)
    {
        int changed = 0;
        CK(cudaMemsetAsync(fs.ctl.p + 2, 0, sizeof(int), st));
        k_fuse_correct<<<blocks_for(static_cast<size_t>(n)), kThreads, 0, st>>>(n, fs.p.voxel_size, fs.keys.p, fs.vals.p, fs.cap - 1, fs.x.p, fs.y.p,
                                                                              fs.z.p, fs.sdf.p, fs.w.p, fs.sdf2.p, fs.w2.p, fs.ctl.p + 2);
        fs.sdf.swap(fs.sdf2); fs.w.swap(fs.w2);
        CK(cudaMemcpyAsync(&changed, fs.ctl.p + 2, sizeof(int), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        tm.phases["fusion_sweeps"].count += 1;
        if (!changed) break;
    }
}

int fusion::sort(FusionState& fs, bool valid_only, cudaStream_t st)
{
    if (fs.n <= 0) return 0;
    const int n = static_cast<int>(fs.n);
    fs.sk.ensure(n); fs.sk2.ensure(n); fs.si.ensure(n); fs.si2.ensure(n);
    CK(cudaMemsetAsync(fs.ctl.p + 3, 0, sizeof(int), st));
    k_fuse_sort_keys<<<blocks_for(n), kThreads, 0, st>>>(n, fs.x.p, fs.y.p, fs.z.p, fs.w.p, valid_only ? 1 : 0, fs.sk.p, fs.si.p, fs.ctl.p + 3);
    size_t bytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, fs.sk.p, fs.sk2.p, fs.si.p, fs.si2.p, n, 0, 64, st));
    fs.cub.ensure(bytes);
    CK(cub::DeviceRadixSort::SortPairs(fs.cub.p, bytes, fs.sk.p, fs.sk2.p, fs.si.p, fs.si2.p, n, 0, 64, st));
    fs.si.swap(fs.si2);                                  // sorted indices now in fs.si
    int m = n;
    if (valid_only) CK(cudaMemcpyAsync(&m, fs.ctl.p + 3, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    return m;
}

void fusion::convert(const FusionState& fs, int m, const VoxelArrays& out, cudaStream_t st)
{
    k_fuse_convert<<<blocks_for(static_cast<size_t>(m)), kThreads, 0, st>>>(m, fs.si.p, fuse_volume(fs), out);
}

FuseView fusion::view(const FusionState& fs)
{
    return FuseView{fs.keys.p, fs.vals.p, fs.cap - 1, fs.x.p, fs.y.p, fs.z.p, fs.sdf.p, fs.w.p, fs.n};
}

void fusion::download(FusionState& fs, int32_t* xyz, float* sdf, float* weight, uint8_t* rgb, cudaStream_t st)
{
    const int64_t n = fs.n;
    if (n <= 0) return;
    sort(fs, false, st);
    const size_t un = static_cast<size_t>(n);
    Dev<int32_t> dxyz; Dev<float> dsdf, dw; Dev<uint8_t> drgb;
    dxyz.ensure(3 * un); dsdf.ensure(un); dw.ensure(un); drgb.ensure(3 * un);
    k_fuse_gather<<<blocks_for(un), kThreads, 0, st>>>(n, fs.si.p, fuse_volume(fs), dxyz.p, dsdf.p, dw.p, drgb.p);
    if (xyz) CK(cudaMemcpyAsync(xyz, dxyz.p, 3 * un * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (sdf) CK(cudaMemcpyAsync(sdf, dsdf.p, un * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (weight) CK(cudaMemcpyAsync(weight, dw.p, un * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (rgb) CK(cudaMemcpyAsync(rgb, drgb.p, 3 * un, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
}

} // namespace i3d
