/*
 * i3d_mesh.cu — the surface extraction: its kernels (i3d_mesh.cuh), the colour modes it can take its colours from (i3d_vis.cuh), their
 * CUB passes and the host code that sequences them (i3d_mesh.h).  Keeping them out of i3d_engine.cu leaves the engine's device module
 * as it is.
 */
#include <climits>
#include <cstdio>

#include "i3d_mesh.cuh"
#include "i3d_vis.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

namespace i3d
{
namespace mesh
{
namespace
{
struct AddI64 { __device__ __forceinline__ int64_t operator()(int64_t a, int64_t b) const { return a + b; } };
struct MaxI32 { __device__ __forceinline__ int32_t operator()(int32_t a, int32_t b) const { return a > b ? a : b; } };

// runs one CUB device call twice: temp-size query, then the call on ms.cub (grown, never shrunk)
template <class Fn>
void cub_call(MeshState& ms, Fn&& fn)
{
    size_t bytes = 0;
    CK(fn(static_cast<void*>(nullptr), bytes));
    ms.cub.ensure(bytes);
    CK(fn(static_cast<void*>(ms.cub.p), bytes));
}

// Device time per stage of one extraction: event pairs around device-only segments, each credited to a stage.  The host round trips
// that read counts back fall between segments, so they are not counted.
struct MeshSegments
{
    MeshState& ms; cudaStream_t st; int used = 0; int stage[8];
    void begin(int s) { CK(cudaEventRecord(ms.ev[2 * used], st)); stage[used] = s; }
    void end() { CK(cudaEventRecord(ms.ev[2 * used + 1], st)); ++used; }
};

template <class T>
T read_back(const T* d, cudaStream_t st)
{
    T h{};
    CK(cudaMemcpyAsync(&h, d, sizeof(T), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return h;
}
} // namespace

void colorize(MeshState& ms, Timing& tm, const GridView& g, const SubvolGrid& sg, const double* sub_sh, int S, int mode, cudaStream_t st)
{
    begin_timing(tm, {"mesh_colorize"});
    ms.vis_rgb.ensure(static_cast<size_t>(g.n));
    {
        Timer t(tm, st, "mesh_colorize");
        uchar4* out = ms.vis_rgb.p;
        const unsigned nb = blocks_for(g.n);
        switch (mode)
        {
        case I3D_MESH_COLOR_NORMALS: k_vis_colors<I3D_MESH_COLOR_NORMALS><<<nb, kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
        case I3D_MESH_COLOR_LAPLACIAN: k_vis_colors<I3D_MESH_COLOR_LAPLACIAN><<<nb, kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
        case I3D_MESH_COLOR_INTENSITY: k_vis_colors<I3D_MESH_COLOR_INTENSITY><<<nb, kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
        case I3D_MESH_COLOR_INTENSITY_GRAD: k_vis_colors<I3D_MESH_COLOR_INTENSITY_GRAD><<<nb, kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
        case I3D_MESH_COLOR_ALBEDO: k_vis_colors<I3D_MESH_COLOR_ALBEDO><<<nb, kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
        case I3D_MESH_COLOR_SHADING_SV: k_vis_colors<I3D_MESH_COLOR_SHADING_SV><<<nb, kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
        case I3D_MESH_COLOR_SHADING_SV_CONST: k_vis_colors<I3D_MESH_COLOR_SHADING_SV_CONST><<<nb, kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
        case I3D_MESH_COLOR_CHROMACITY: k_vis_colors<I3D_MESH_COLOR_CHROMACITY><<<nb, kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
        default: break;
        }
    }
    collect_kernel_times(tm, st);
    CK(cudaGetLastError());
}

int extract(MeshState& ms, const MeshGrid& g, bool largest_component_only, I3DMeshInfo* info, std::string& error, cudaStream_t st)
{
    const int64_t n = g.n;
    ms.have_mesh = false;
    if (!ms.ev_ready) { for (auto& ev : ms.ev) CK(cudaEventCreate(&ev)); ms.ev_ready = true; }
    I3DMeshInfo inf{};

    enum { CLASSIFY, EMIT, WELD, CLEAN, COMPONENTS };
    MeshSegments seg{ms, st};

    // 1. cube cases and per-voxel triangle counts -> face offsets (int64 exclusive scan of the counts)
    ms.cases.ensure(n); ms.cnt.ensure(n); ms.off.ensure(n); ms.cubes.ensure(1); ms.sel.ensure(1); ms.best.ensure(1);
    seg.begin(CLASSIFY);
    CK(cudaMemsetAsync(ms.cubes.p, 0, sizeof(unsigned long long), st));
    k_mesh_classify<<<blocks_for(n), kThreads, 0, st>>>(g, ms.cases.p, ms.cnt.p, ms.cubes.p);
    cub_call(ms, [&](void* t, size_t& b) {
        return cub::DeviceScan::ExclusiveScan(t, b, static_cast<const int32_t*>(ms.cnt.p), ms.off.p, AddI64(), static_cast<int64_t>(0), static_cast<int>(n), st);
    });
    seg.end();
    inf.num_cubes = static_cast<int64_t>(read_back(ms.cubes.p, st));
    const int64_t F0 = read_back(ms.off.p + (n - 1), st) + read_back(ms.cnt.p + (n - 1), st);
    inf.num_faces_raw = F0;
    // corner and vertex ids are int32 (as the PLY's indices); element offsets into the interleaved arrays are computed in int64
    if (3 * F0 > INT_MAX)
    {
        error = "i3d_extract_mesh: " + std::to_string(static_cast<long long>(F0)) + " triangles exceed the int32 corner indices of the mesh";
        return 1;
    }
    const int32_t M = static_cast<int32_t>(3 * F0);
    float* vpos = nullptr; uint8_t* vcol = nullptr; int3* faces = nullptr;
    int64_t V = 0, F = 0;
    if (M > 0)
    {
        // 2. the triangle soup, corner by corner
        ms.cpos.ensure(3 * static_cast<size_t>(M)); ms.ccol.ensure(3 * static_cast<size_t>(M));
        ms.klo.ensure(M); ms.klo2.ensure(M); ms.khi.ensure(M); ms.khi2.ensure(M); ms.perm.ensure(M); ms.perm2.ensure(M);
        seg.begin(EMIT);
        k_mesh_emit<<<blocks_for(n), kThreads, 0, st>>>(g, ms.cases.p, ms.cnt.p, ms.off.p, MeshCorners{ms.cpos.p, ms.ccol.p, ms.klo.p, ms.khi.p});
        seg.end();

        // 3. welding: stable sort of the corner indices by position (z bits, then x|y bits), segment heads, ids by first appearance
        ms.first.ensure(M); ms.fid.ensure(M); ms.head.ensure(M); ms.seg.ensure(M); ms.cvid.ensure(M);
        seg.begin(WELD);
        k_mesh_iota<<<blocks_for(M), kThreads, 0, st>>>(M, ms.perm2.p);
        cub_call(ms, [&](void* t, size_t& b) {
            return cub::DeviceRadixSort::SortPairs(t, b, static_cast<const uint32_t*>(ms.klo.p), ms.klo2.p, static_cast<const int32_t*>(ms.perm2.p), ms.perm.p,
                                                   M, 0, 32, st);
        });
        k_gather_key_hi<<<blocks_for(M), kThreads, 0, st>>>(M, ms.perm.p, ms.khi.p, ms.khi2.p);
        cub_call(ms, [&](void* t, size_t& b) {
            return cub::DeviceRadixSort::SortPairs(t, b, static_cast<const unsigned long long*>(ms.khi2.p), ms.khi.p, static_cast<const int32_t*>(ms.perm.p),
                                                   ms.perm2.p, M, 0, 64, st);
        });
        k_weld_heads<<<blocks_for(M), kThreads, 0, st>>>(M, ms.perm2.p, ms.khi.p, ms.klo.p, ms.first.p, ms.head.p);
        cub_call(ms, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, static_cast<const int32_t*>(ms.first.p), ms.fid.p, M, st); });
        cub_call(ms, [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveScan(t, b, static_cast<const int32_t*>(ms.head.p), ms.seg.p, MaxI32(), M, st); });
        seg.end();
        const int64_t Vw = read_back(ms.fid.p + (M - 1), st) + read_back(ms.first.p + (M - 1), st);
        ms.vpos.ensure(3 * static_cast<size_t>(Vw)); ms.vcol.ensure(3 * static_cast<size_t>(Vw));
        seg.begin(WELD);
        k_weld_assign<<<blocks_for(M), kThreads, 0, st>>>(M, ms.perm2.p, ms.seg.p, ms.fid.p, ms.cpos.p, ms.ccol.p, ms.cvid.p, ms.vpos.p, ms.vcol.p);
        seg.end();
        inf.num_vertices_welded = Vw;

        // 4. degenerate faces, survivors kept in order; the vertices stay
        const int32_t F0i = static_cast<int32_t>(F0);
        const int3* faces0 = reinterpret_cast<const int3*>(ms.cvid.p);
        ms.keep.ensure(F0); ms.faces.ensure(F0);
        seg.begin(CLEAN);
        k_face_clean<<<blocks_for(F0i), kThreads, 0, st>>>(F0i, faces0, ms.vpos.p, ms.keep.p);
        cub_call(ms, [&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, faces0, static_cast<const uint8_t*>(ms.keep.p), ms.faces.p, ms.sel.p, F0i, st); });
        seg.end();
        const int32_t F1 = read_back(ms.sel.p, st);
        inf.num_faces_clean = F1;
        vpos = ms.vpos.p; vcol = ms.vcol.p; faces = ms.faces.p; V = Vw; F = F1;

        // 5. the largest face-connected component, then only the vertices it uses
        if (largest_component_only)
        {
            const int32_t Vi = static_cast<int32_t>(Vw);
            ms.parent.ensure(Vw); ms.ccount.ensure(Vw); ms.cminf.ensure(Vw); ms.used.ensure(Vw); ms.newid.ensure(Vw);
            ms.faces2.ensure(std::max<int32_t>(F1, 1));
            int32_t F2 = 0, V2 = 0;
            if (F1 > 0)
            {
                seg.begin(COMPONENTS);
                k_mesh_iota<<<blocks_for(Vi), kThreads, 0, st>>>(Vi, ms.parent.p);
                k_cc_union<<<blocks_for(F1), kThreads, 0, st>>>(F1, ms.faces.p, ms.parent.p);
                k_cc_flatten<<<blocks_for(Vi), kThreads, 0, st>>>(Vi, ms.parent.p);
                CK(cudaMemsetAsync(ms.ccount.p, 0, Vw * sizeof(unsigned), st));
                CK(cudaMemsetAsync(ms.cminf.p, 0xFF, Vw * sizeof(unsigned), st));
                CK(cudaMemsetAsync(ms.best.p, 0, sizeof(unsigned long long), st));
                k_cc_count<<<blocks_for(F1), kThreads, 0, st>>>(F1, ms.faces.p, ms.parent.p, ms.ccount.p, ms.cminf.p);
                k_cc_best<<<blocks_for(Vi), kThreads, 0, st>>>(Vi, ms.ccount.p, ms.cminf.p, ms.best.p);
                k_cc_keep<<<blocks_for(F1), kThreads, 0, st>>>(F1, ms.faces.p, ms.parent.p, ms.best.p, ms.keep.p);
                cub_call(ms, [&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, static_cast<const int3*>(ms.faces.p), static_cast<const uint8_t*>(ms.keep.p), ms.faces2.p, ms.sel.p, F1, st); });
                seg.end();
                F2 = read_back(ms.sel.p, st);
                seg.begin(COMPONENTS);
                CK(cudaMemsetAsync(ms.used.p, 0, Vw * sizeof(int32_t), st));
                if (F2 > 0) k_mark_used<<<blocks_for(F2), kThreads, 0, st>>>(F2, ms.faces2.p, ms.used.p);
                cub_call(ms, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, static_cast<const int32_t*>(ms.used.p), ms.newid.p, Vi, st); });
                seg.end();
                V2 = read_back(ms.newid.p + (Vi - 1), st) + read_back(ms.used.p + (Vi - 1), st);
                ms.vpos2.ensure(3 * static_cast<size_t>(V2)); ms.vcol2.ensure(3 * static_cast<size_t>(V2));
                seg.begin(COMPONENTS);
                k_compact_vertices<<<blocks_for(Vi), kThreads, 0, st>>>(Vi, ms.used.p, ms.newid.p, ms.vpos.p, ms.vcol.p, ms.vpos2.p, ms.vcol2.p);
                if (F2 > 0) k_remap_faces<<<blocks_for(F2), kThreads, 0, st>>>(F2, ms.newid.p, ms.faces2.p);
                seg.end();
            }
            vpos = ms.vpos2.p; vcol = ms.vcol2.p; faces = ms.faces2.p; V = V2; F = F2;
        }
    }
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    double t_ms[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int k = 0; k < seg.used; ++k)
    {
        float t = 0.f;
        CK(cudaEventElapsedTime(&t, ms.ev[2 * k], ms.ev[2 * k + 1]));
        t_ms[seg.stage[k]] += t;
    }
    inf.ms_classify = t_ms[CLASSIFY]; inf.ms_emit = t_ms[EMIT]; inf.ms_weld = t_ms[WELD]; inf.ms_clean = t_ms[CLEAN]; inf.ms_components = t_ms[COMPONENTS];
    inf.num_faces = F; inf.num_vertices = V;
    ms.mesh_vpos = vpos; ms.mesh_vcol = vcol; ms.mesh_faces = faces; ms.mesh_V = V; ms.mesh_F = F;
    ms.have_mesh = true;
    if (info) *info = inf;
    return 0;
}

int simplify(MeshState& ms, float cell_size, I3DSimplifyInfo* info, std::string& error, cudaStream_t st)
{
    if (!ms.ev_ready) { for (auto& ev : ms.ev) CK(cudaEventCreate(&ev)); ms.ev_ready = true; }
    const int32_t V = static_cast<int32_t>(ms.mesh_V), F = static_cast<int32_t>(ms.mesh_F);
    const float* vpos = ms.mesh_vpos; const uint8_t* vcol = ms.mesh_vcol; const int3* faces = ms.mesh_faces;
    // the output slot the resident mesh is not in
    const int out = (ms.mesh_vpos == ms.s_vpos[0].p || ms.mesh_faces == ms.s_faces[0].p) ? 1 : 0;
    I3DSimplifyInfo inf{};

    enum { CLUSTER, QUADRICS, REPRESENTATIVES, FACES, COMPACT };
    MeshSegments seg{ms, st};

    // 1. cells, then clusters numbered by first appearance over the vertex ids: the welding's two stable radix passes (z, then x|y), its
    //    segment heads and scans, and the cluster id of every vertex.  The cell check is read back with the cluster count, before
    //    anything but scratch has been written.
    int32_t K = 0;
    if (V > 0)
    {
        ms.s_bad.ensure(1); ms.klo.ensure(V); ms.klo2.ensure(V); ms.khi.ensure(V); ms.khi2.ensure(V); ms.perm.ensure(V); ms.perm2.ensure(V);
        ms.first.ensure(V); ms.fid.ensure(V); ms.head.ensure(V); ms.seg.ensure(V); ms.s_cid.ensure(V); ms.s_run.ensure(V);
        seg.begin(CLUSTER);
        CK(cudaMemsetAsync(ms.s_bad.p, 0, sizeof(int32_t), st));
        k_simp_cell_keys<<<blocks_for(V), kThreads, 0, st>>>(V, vpos, cell_size, ms.klo.p, ms.khi.p, ms.s_bad.p);
        k_mesh_iota<<<blocks_for(V), kThreads, 0, st>>>(V, ms.perm2.p);
        cub_call(ms, [&](void* t, size_t& b) {
            return cub::DeviceRadixSort::SortPairs(t, b, static_cast<const uint32_t*>(ms.klo.p), ms.klo2.p, static_cast<const int32_t*>(ms.perm2.p), ms.perm.p,
                                                   V, 0, 32, st);
        });
        k_gather_key_hi<<<blocks_for(V), kThreads, 0, st>>>(V, ms.perm.p, ms.khi.p, ms.khi2.p);
        cub_call(ms, [&](void* t, size_t& b) {
            return cub::DeviceRadixSort::SortPairs(t, b, static_cast<const unsigned long long*>(ms.khi2.p), ms.khi.p, static_cast<const int32_t*>(ms.perm.p),
                                                   ms.perm2.p, V, 0, 64, st);
        });
        k_weld_heads<<<blocks_for(V), kThreads, 0, st>>>(V, ms.perm2.p, ms.khi.p, ms.klo.p, ms.first.p, ms.head.p);
        cub_call(ms, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, static_cast<const int32_t*>(ms.first.p), ms.fid.p, V, st); });
        cub_call(ms, [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveScan(t, b, static_cast<const int32_t*>(ms.head.p), ms.seg.p, MaxI32(), V, st); });
        k_simp_cluster_ids<<<blocks_for(V), kThreads, 0, st>>>(V, ms.perm2.p, ms.seg.p, ms.fid.p, ms.s_cid.p, ms.s_run.p);
        seg.end();
        if (read_back(ms.s_bad.p, st))
        {
            char buf[160];
            std::snprintf(buf, sizeof(buf), "i3d_simplify_mesh: cell_size %g puts a vertex in a cell whose coordinate is not finite or outside int32",
                          static_cast<double>(cell_size));
            error = buf;
            return 1;
        }
        K = read_back(ms.fid.p + (V - 1), st) + read_back(ms.first.p + (V - 1), st);
    }
    inf.num_clusters = K;
    // bits of the largest cluster id, for the radix passes over cluster ids
    int nb = 1;
    while (nb < 31 && (static_cast<int64_t>(1) << nb) < K) ++nb;

    int32_t F2 = 0, V2 = 0;
    ms.s_faces[out].ensure(F); ms.s_vpos[out].ensure(3 * static_cast<size_t>(K)); ms.s_vcol[out].ensure(3 * static_cast<size_t>(K));
    if (F > 0)
    {
        // 2. the area-weighted plane quadric of every face
        ms.s_quad.ensure(9 * static_cast<size_t>(F));
        seg.begin(QUADRICS);
        k_simp_face_quadrics<<<blocks_for(F), kThreads, 0, st>>>(F, faces, vpos, ms.s_quad.p);
        seg.end();

        // 3. the corners grouped by cluster (stable radix sort: corner order within a cluster), then one thread per cluster sums its
        //    members and its corners' quadrics in order and places its representative
        const int32_t M = 3 * F;
        ms.s_ckey.ensure(M); ms.s_ckey2.ensure(M); ms.s_corner.ensure(M); ms.s_corner2.ensure(M);
        ms.s_cstart.ensure(K); ms.s_cend.ensure(K); ms.s_rpos.ensure(3 * static_cast<size_t>(K)); ms.s_rcol.ensure(3 * static_cast<size_t>(K));
        seg.begin(REPRESENTATIVES);
        k_simp_corner_keys<<<blocks_for(M), kThreads, 0, st>>>(M, reinterpret_cast<const int32_t*>(faces), ms.s_cid.p, ms.s_ckey.p, ms.s_corner.p);
        cub_call(ms, [&](void* t, size_t& b) {
            return cub::DeviceRadixSort::SortPairs(t, b, static_cast<const uint32_t*>(ms.s_ckey.p), ms.s_ckey2.p, static_cast<const int32_t*>(ms.s_corner.p),
                                                   ms.s_corner2.p, M, 0, nb, st);
        });
        CK(cudaMemsetAsync(ms.s_cstart.p, 0, K * sizeof(int32_t), st));
        CK(cudaMemsetAsync(ms.s_cend.p, 0, K * sizeof(int32_t), st));
        k_simp_corner_runs<<<blocks_for(M), kThreads, 0, st>>>(M, ms.s_ckey2.p, ms.s_cstart.p, ms.s_cend.p);
        const SimplifyClusters cl{ms.perm2.p, ms.seg.p, ms.s_run.p, ms.s_corner2.p, ms.s_cstart.p, ms.s_cend.p};
        k_simp_representatives<<<blocks_for(K), kThreads, 0, st>>>(V, K, cl, vpos, vcol, F, ms.s_quad.p, ms.s_rpos.p, ms.s_rcol.p);
        seg.end();

        // 4. faces on cluster ids: collapsed and duplicate faces (stable radix passes over the rotation key), then k_face_clean at the
        //    representatives; the survivors in input order
        ms.s_cfaces.ensure(F); ms.klo.ensure(F); ms.klo2.ensure(F); ms.khi.ensure(F); ms.khi2.ensure(F); ms.perm.ensure(F); ms.perm2.ensure(F);
        ms.keep.ensure(F); ms.sel.ensure(1); ms.s_counts.ensure(2);
        seg.begin(FACES);
        k_simp_face_keys<<<blocks_for(F), kThreads, 0, st>>>(F, faces, ms.s_cid.p, nb, ms.s_cfaces.p, ms.klo.p, ms.khi.p);
        k_mesh_iota<<<blocks_for(F), kThreads, 0, st>>>(F, ms.perm2.p);
        cub_call(ms, [&](void* t, size_t& b) {
            return cub::DeviceRadixSort::SortPairs(t, b, static_cast<const uint32_t*>(ms.klo.p), ms.klo2.p, static_cast<const int32_t*>(ms.perm2.p), ms.perm.p,
                                                   F, 0, nb, st);
        });
        k_gather_key_hi<<<blocks_for(F), kThreads, 0, st>>>(F, ms.perm.p, ms.khi.p, ms.khi2.p);
        cub_call(ms, [&](void* t, size_t& b) {
            return cub::DeviceRadixSort::SortPairs(t, b, static_cast<const unsigned long long*>(ms.khi2.p), ms.khi.p, static_cast<const int32_t*>(ms.perm.p),
                                                   ms.perm2.p, F, 0, 2 * nb, st);
        });
        k_face_clean<<<blocks_for(F), kThreads, 0, st>>>(F, ms.s_cfaces.p, ms.s_rpos.p, ms.keep.p);
        CK(cudaMemsetAsync(ms.s_counts.p, 0, 2 * sizeof(unsigned long long), st));
        k_simp_face_dups<<<blocks_for(F), kThreads, 0, st>>>(F, ms.perm2.p, ms.khi.p, ms.klo.p, ms.s_cfaces.p, ms.keep.p, ms.s_counts.p);
        cub_call(ms, [&](void* t, size_t& b) {
            return cub::DeviceSelect::Flagged(t, b, static_cast<const int3*>(ms.s_cfaces.p), static_cast<const uint8_t*>(ms.keep.p), ms.s_faces[out].p, ms.sel.p, F, st);
        });
        seg.end();
        F2 = read_back(ms.sel.p, st);
        inf.num_faces_collapsed = static_cast<int64_t>(read_back(ms.s_counts.p, st));
        inf.num_faces_duplicate = static_cast<int64_t>(read_back(ms.s_counts.p + 1, st));
        inf.num_faces_degenerate = F - F2 - inf.num_faces_collapsed - inf.num_faces_duplicate;

        // 5. only the clusters the surviving faces use, in order, and the faces renumbered
        ms.used.ensure(K); ms.newid.ensure(K);
        seg.begin(COMPACT);
        CK(cudaMemsetAsync(ms.used.p, 0, K * sizeof(int32_t), st));
        if (F2 > 0) k_mark_used<<<blocks_for(F2), kThreads, 0, st>>>(F2, ms.s_faces[out].p, ms.used.p);
        cub_call(ms, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, static_cast<const int32_t*>(ms.used.p), ms.newid.p, K, st); });
        k_compact_vertices<<<blocks_for(K), kThreads, 0, st>>>(K, ms.used.p, ms.newid.p, ms.s_rpos.p, ms.s_rcol.p, ms.s_vpos[out].p, ms.s_vcol[out].p);
        if (F2 > 0) k_remap_faces<<<blocks_for(F2), kThreads, 0, st>>>(F2, ms.newid.p, ms.s_faces[out].p);
        seg.end();
        V2 = read_back(ms.newid.p + (K - 1), st) + read_back(ms.used.p + (K - 1), st);
    }
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    double t_ms[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int k = 0; k < seg.used; ++k)
    {
        float t = 0.f;
        CK(cudaEventElapsedTime(&t, ms.ev[2 * k], ms.ev[2 * k + 1]));
        t_ms[seg.stage[k]] += t;
    }
    inf.ms_cluster = t_ms[CLUSTER]; inf.ms_quadrics = t_ms[QUADRICS]; inf.ms_representatives = t_ms[REPRESENTATIVES]; inf.ms_faces = t_ms[FACES];
    inf.ms_compact = t_ms[COMPACT];
    inf.num_faces = F2; inf.num_vertices = V2;
    ms.mesh_vpos = ms.s_vpos[out].p; ms.mesh_vcol = ms.s_vcol[out].p; ms.mesh_faces = ms.s_faces[out].p; ms.mesh_V = V2; ms.mesh_F = F2;
    if (info) *info = inf;
    return 0;
}

} // namespace mesh
} // namespace i3d
