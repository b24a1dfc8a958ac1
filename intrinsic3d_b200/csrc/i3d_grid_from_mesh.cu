/*
 * i3d_grid_from_mesh.cu — the voxel grid from a triangle mesh: its kernels (i3d_grid_from_mesh.cuh) and the host code that sequences them
 * (i3d_grid_from_mesh.h).  The search grid is the distance module's (distance::plan / build).
 */
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "i3d_grid_from_mesh.cuh"
#include "i3d_grid_from_mesh.h"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

namespace i3d
{
namespace gfm
{
namespace
{
std::string format(const char* fmt, ...)
{
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    return buf;
}

template <class K>
void sort_pairs(GridFromMeshState& s, K*& k, K*& k2, int32_t*& v, int32_t*& v2, int64_t n, int end_bit, cudaStream_t st)
{
    size_t bytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, k, k2, v, v2, n, 0, end_bit, st));
    s.cub.ensure(bytes);
    CK(cub::DeviceRadixSort::SortPairs(s.cub.p, bytes, k, k2, v, v2, n, 0, end_bit, st));
    std::swap(k, k2); std::swap(v, v2);
}

unsigned long long read_counter(GridFromMeshState& s, int slot, cudaStream_t st)
{
    unsigned long long v = 0;
    CK(cudaMemcpyAsync(&v, s.counters.p + slot, sizeof(v), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return v;
}
} // namespace

int query(GridFromMeshState& s, const DistMesh& m, const I3DGridFromMeshParams& p, I3DGridFromMeshInfo& info, std::string& error, cudaStream_t st)
{
    if (!s.ev_ready) { for (auto& ev : s.ev) CK(cudaEventCreate(&ev)); s.ev_ready = true; }
    std::memset(&info, 0, sizeof(info));
    const float vs = p.voxel_size, b = p.band * p.voxel_size;          // FM(band, voxel_size)
    GfmConst C;
    C.voxel_size = vs; C.b = b;
    const float r = b + static_cast<float>(3.5 * std::sqrt(3.0) + 1.0) * vs;
    C.r2 = r * r;
    C.inv_voxel_size_d = 1.0 / static_cast<double>(vs); C.b_d = static_cast<double>(b);
    s.counters.ensure(GFM_COUNTERS);
    CK(cudaMemsetAsync(s.counters.p, 0, GFM_COUNTERS * sizeof(unsigned long long), st));

    // the search grid is sized first: its caps and the lattice range refuse before anything else runs
    DistGrid g;
    int64_t entries = 0;
    double bounds[6];
    if (!distance::plan(s.grid, m, p.cell_size, b, g, entries, bounds, error, st)) return 1;
    const double lim = static_cast<double>((1 << 20) - 8);
    for (int k = 0; k < 3; ++k)
    {
        const double c0 = std::floor((bounds[k] - b) / vs), c1 = std::ceil((bounds[3 + k] + b) / vs);
        if (!(c0 >= -lim && c1 <= lim))
            return error = format("the band around the mesh spans lattice coordinates [%.0f, %.0f] on axis %d at voxel_size %g, outside +-%.0f", c0, c1, k,
                                  static_cast<double>(vs), lim), 1;
    }
    const int64_t V = m.V, F = m.F, n3 = 3 * F;
    const unsigned nbf = blocks_for(static_cast<size_t>(F));
    k_gfm_brick_pairs<<<nbf, kThreads, 0, st>>>(m, C, s.counters.p);
    const long long pairs = static_cast<long long>(read_counter(s, GFM_PAIRS, st));
    if (pairs > I3D_GRID_FROM_MESH_MAX_PAIRS)
        return error = format("%lld (face, brick) pairs exceed I3D_GRID_FROM_MESH_MAX_PAIRS (%lld): a face spans too many bricks at voxel_size %g", pairs,
                              static_cast<long long>(I3D_GRID_FROM_MESH_MAX_PAIRS), static_cast<double>(vs)), 1;

    // candidate bricks: the keys of every (face, brick) pair that passes, sorted and made unique
    CK(cudaEventRecord(s.ev[0], st));
    s.bk.ensure(static_cast<size_t>(pairs)); s.bk2.ensure(static_cast<size_t>(pairs)); s.nsel.ensure(1);
    k_gfm_brick_fill<<<nbf, kThreads, 0, st>>>(m, C, s.bk.p, s.counters.p);
    CK(cudaEventRecord(s.ev[1], st));
    const int64_t filled = static_cast<int64_t>(read_counter(s, GFM_FILL, st));
    int64_t nb = 0;
    if (filled > 0)
    {
        size_t bytes = 0;
        CK(cub::DeviceRadixSort::SortKeys(nullptr, bytes, s.bk.p, s.bk2.p, filled, 10, 64, st));
        s.cub.ensure(bytes);
        CK(cub::DeviceRadixSort::SortKeys(s.cub.p, bytes, s.bk.p, s.bk2.p, filled, 10, 64, st));
        bytes = 0;
        CK(cub::DeviceSelect::Unique(nullptr, bytes, s.bk2.p, s.bk.p, s.nsel.p, filled, st));
        s.cub.ensure(bytes);
        CK(cub::DeviceSelect::Unique(s.cub.p, bytes, s.bk2.p, s.bk.p, s.nsel.p, filled, st));
        CK(cudaMemcpyAsync(&nb, s.nsel.p, sizeof(nb), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    }
    CK(cudaEventRecord(s.ev[2], st));
    const int64_t nc = 512 * nb;
    if (nc > I3D_GRID_FROM_MESH_MAX_VOXELS)
        return error = format("%lld candidate voxels exceed I3D_GRID_FROM_MESH_MAX_VOXELS (%lld)", static_cast<long long>(nc),
                              static_cast<long long>(I3D_GRID_FROM_MESH_MAX_VOXELS)), 1;

    // welding and pseudonormals
    s.wk32.ensure(V); s.wk32b.ensure(V); s.wk64.ensure(V); s.wk64b.ensure(V); s.wi.ensure(V); s.wi2.ensure(V); s.weld.ensure(V); s.vb.ensure(V);
    s.vk.ensure(n3); s.vk2.ensure(n3); s.ek.ensure(n3); s.ek2.ensure(n3); s.vi.ensure(n3); s.vi2.ensure(n3); s.ei.ensure(n3); s.ei2.ensure(n3);
    s.fn.ensure(3 * F); s.vn.ensure(3 * n3); s.en.ensure(3 * n3); s.eb.ensure(n3);
    const unsigned nbv = blocks_for(static_cast<size_t>(V)), nb3 = blocks_for(static_cast<size_t>(n3));
    CK(cudaEventRecord(s.ev[3], st));
    {
        uint32_t *k32 = s.wk32.p, *k32b = s.wk32b.p;
        unsigned long long *k64 = s.wk64.p, *k64b = s.wk64b.p;
        int32_t *a = s.wi.p, *a2 = s.wi2.p;
        k_gfm_weld_z<<<nbv, kThreads, 0, st>>>(V, m.vpos, k32, a);
        sort_pairs(s, k32, k32b, a, a2, V, 32, st);
        k_gfm_weld_xy<<<nbv, kThreads, 0, st>>>(V, m.vpos, a, k64);
        sort_pairs(s, k64, k64b, a, a2, V, 64, st);
        k_gfm_weld_runs<<<nbv, kThreads, 0, st>>>(V, m.vpos, a, s.weld.p, s.counters.p);
    }
    k_gfm_face_normals<<<nbf, kThreads, 0, st>>>(m, s.fn.p);
    {
        uint32_t *vk = s.vk.p, *vk2 = s.vk2.p;
        unsigned long long *ek = s.ek.p, *ek2 = s.ek2.p;
        int32_t *vi = s.vi.p, *vi2 = s.vi2.p, *ei = s.ei.p, *ei2 = s.ei2.p;
        k_gfm_incidences<<<nb3, kThreads, 0, st>>>(m, s.weld.p, vk, vi, ek, ei);
        sort_pairs(s, vk, vk2, vi, vi2, n3, 32, st);
        sort_pairs(s, ek, ek2, ei, ei2, n3, 64, st);
        CK(cudaMemsetAsync(s.vb.p, 0, static_cast<size_t>(V), st));
        k_gfm_vertex_normals<<<nb3, kThreads, 0, st>>>(m, vk, vi, s.fn.p, s.vn.p);
        k_gfm_edge_normals<<<nb3, kThreads, 0, st>>>(F, ek, ei, s.fn.p, s.en.p, s.eb.p, s.vb.p, s.counters.p);
    }
    CK(cudaEventRecord(s.ev[4], st));
    distance::build(s.grid, m, g, entries, st);
    CK(cudaEventRecord(s.ev[5], st));

    // the query
    s.keep.ensure(nc); s.sdf.ensure(nc); s.face.ensure(nc); s.feat.ensure(nc);
    CK(cudaEventRecord(s.ev[6], st));
    if (nc > 0)
        k_gfm_query<<<blocks_for(static_cast<size_t>(nc)), kThreads, 0, st>>>(nc, s.bk.p, m, g, C, GfmTopology{s.fn.p, s.vn.p, s.en.p, s.eb.p, s.vb.p, s.weld.p},
                                                                             s.keep.p, s.sdf.p, s.face.p, s.feat.p, s.counters.p);
    CK(cudaEventRecord(s.ev[7], st));
    unsigned long long cnt[GFM_COUNTERS];
    CK(cudaMemcpyAsync(cnt, s.counters.p, sizeof(cnt), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    auto ms = [](cudaEvent_t a, cudaEvent_t c) { float t = 0.f; CK(cudaEventElapsedTime(&t, a, c)); return static_cast<double>(t); };
    info.num_faces = F;
    info.num_vertices_welded = static_cast<int64_t>(cnt[GFM_WELDED]);
    info.num_boundary_edges = static_cast<int64_t>(cnt[GFM_BOUNDARY]);
    info.num_brick_pairs = pairs;
    info.num_candidate_bricks = nb; info.num_candidate_voxels = nc;
    info.num_voxels = static_cast<int64_t>(cnt[GFM_EMITTED]); info.num_negative = static_cast<int64_t>(cnt[GFM_NEGATIVE]);
    info.num_beyond_band = static_cast<int64_t>(cnt[GFM_BEYOND]);
    info.num_dropped_rim = static_cast<int64_t>(cnt[GFM_RIM]);
    info.num_dropped_zero_normal = static_cast<int64_t>(cnt[GFM_ZERO_NORMAL]);
    info.num_dropped_zero_dot = static_cast<int64_t>(cnt[GFM_ZERO_DOT]);
    info.point_triangle_tests = static_cast<int64_t>(cnt[GFM_TESTS]);
    info.cell_size = g.h;
    for (int k = 0; k < 3; ++k) info.grid[k] = g.n[k];
    info.ms_bricks = ms(s.ev[0], s.ev[2]);
    info.ms_topology = ms(s.ev[3], s.ev[4]);
    info.ms_grid = ms(s.ev[4], s.ev[5]);
    info.ms_query = ms(s.ev[6], s.ev[7]);
    s.num_bricks = nb;
    return 0;
}

void gather(GridFromMeshState& s, const int32_t* act, int64_t m, const VoxelArrays& out, cudaStream_t st)
{
    s.last_face.ensure(static_cast<size_t>(m)); s.last_feat.ensure(static_cast<size_t>(m));
    k_gfm_gather<<<blocks_for(static_cast<size_t>(m)), kThreads, 0, st>>>(m, act, s.bk.p, s.sdf.p, s.face.p, s.feat.p, out, s.last_face.p, s.last_feat.p);
    s.last_n = m; s.have_last = true;
}

} // namespace gfm
} // namespace i3d
