/*
 * i3d_mesh.cu — the surface-extraction kernels (i3d_mesh.cuh), the colour modes they can take their colours from (i3d_vis.cuh) and
 * their CUB passes, compiled as a translation unit of their own, and the host wrappers of i3d_mesh.h that launch them.  Keeping them
 * out of i3d_engine.cu leaves the engine's device module as it is.
 */
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
inline unsigned blocks(int64_t n) { return static_cast<unsigned>((n + kThreads - 1) / kThreads); }
} // namespace

void colorize(const GridView& g, const SubvolGrid& sg, const double* sub_sh, int S, int mode, uchar4* out, cudaStream_t st)
{
    switch (mode)
    {
    case I3D_MESH_COLOR_NORMALS: k_vis_colors<I3D_MESH_COLOR_NORMALS><<<blocks(g.n), kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
    case I3D_MESH_COLOR_LAPLACIAN: k_vis_colors<I3D_MESH_COLOR_LAPLACIAN><<<blocks(g.n), kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
    case I3D_MESH_COLOR_INTENSITY: k_vis_colors<I3D_MESH_COLOR_INTENSITY><<<blocks(g.n), kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
    case I3D_MESH_COLOR_INTENSITY_GRAD: k_vis_colors<I3D_MESH_COLOR_INTENSITY_GRAD><<<blocks(g.n), kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
    case I3D_MESH_COLOR_ALBEDO: k_vis_colors<I3D_MESH_COLOR_ALBEDO><<<blocks(g.n), kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
    case I3D_MESH_COLOR_SHADING_SV: k_vis_colors<I3D_MESH_COLOR_SHADING_SV><<<blocks(g.n), kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
    case I3D_MESH_COLOR_SHADING_SV_CONST: k_vis_colors<I3D_MESH_COLOR_SHADING_SV_CONST><<<blocks(g.n), kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
    case I3D_MESH_COLOR_CHROMACITY: k_vis_colors<I3D_MESH_COLOR_CHROMACITY><<<blocks(g.n), kThreads, 0, st>>>(g, sg, sub_sh, S, out); break;
    default: break;     // the engine validates the mode before it calls
    }
}

void classify(const MeshGrid& g, uint8_t* cube_case, int32_t* tri_count, unsigned long long* num_cubes, cudaStream_t st)
{
    k_mesh_classify<<<blocks(g.n), kThreads, 0, st>>>(g, cube_case, tri_count, num_cubes);
}
cudaError_t face_offsets(void* tmp, size_t& bytes, const int32_t* tri_count, int64_t* face_off, int n, cudaStream_t st)
{
    return cub::DeviceScan::ExclusiveScan(tmp, bytes, tri_count, face_off, AddI64(), static_cast<int64_t>(0), n, st);
}
void emit(const MeshGrid& g, const uint8_t* cube_case, const int32_t* tri_count, const int64_t* face_off, const MeshCorners& out, cudaStream_t st)
{
    k_mesh_emit<<<blocks(g.n), kThreads, 0, st>>>(g, cube_case, tri_count, face_off, out);
}
void iota(int32_t m, int32_t* out, cudaStream_t st) { k_mesh_iota<<<blocks(m), kThreads, 0, st>>>(m, out); }
cudaError_t sort_z(void* tmp, size_t& bytes, const uint32_t* key_lo, uint32_t* key_lo_sorted, const int32_t* perm_in, int32_t* perm_out, int32_t m,
                   cudaStream_t st)
{
    return cub::DeviceRadixSort::SortPairs(tmp, bytes, key_lo, key_lo_sorted, perm_in, perm_out, m, 0, 32, st);
}
void gather_key_hi(int32_t m, const int32_t* perm, const unsigned long long* key_hi, unsigned long long* out, cudaStream_t st)
{
    k_gather_key_hi<<<blocks(m), kThreads, 0, st>>>(m, perm, key_hi, out);
}
cudaError_t sort_xy(void* tmp, size_t& bytes, const unsigned long long* key_hi, unsigned long long* key_hi_sorted, const int32_t* perm_in,
                    int32_t* perm_out, int32_t m, cudaStream_t st)
{
    return cub::DeviceRadixSort::SortPairs(tmp, bytes, key_hi, key_hi_sorted, perm_in, perm_out, m, 0, 64, st);
}
void weld_heads(int32_t m, const int32_t* perm, const unsigned long long* hi_sorted, const uint32_t* key_lo, int32_t* is_first, int32_t* head_pos,
                cudaStream_t st)
{
    k_weld_heads<<<blocks(m), kThreads, 0, st>>>(m, perm, hi_sorted, key_lo, is_first, head_pos);
}
cudaError_t exclusive_sum(void* tmp, size_t& bytes, const int32_t* in, int32_t* out, int32_t m, cudaStream_t st)
{
    return cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, m, st);
}
cudaError_t inclusive_max(void* tmp, size_t& bytes, const int32_t* in, int32_t* out, int32_t m, cudaStream_t st)
{
    return cub::DeviceScan::InclusiveScan(tmp, bytes, in, out, MaxI32(), m, st);
}
void weld_assign(int32_t m, const int32_t* perm, const int32_t* seg_head, const int32_t* first_id, const float* cpos, const uint8_t* ccol,
                 int32_t* corner_vid, float* vpos, uint8_t* vcol, cudaStream_t st)
{
    k_weld_assign<<<blocks(m), kThreads, 0, st>>>(m, perm, seg_head, first_id, cpos, ccol, corner_vid, vpos, vcol);
}
void face_clean(int32_t f, const int3* faces, const float* vpos, uint8_t* keep, cudaStream_t st)
{
    k_face_clean<<<blocks(f), kThreads, 0, st>>>(f, faces, vpos, keep);
}
cudaError_t select_faces(void* tmp, size_t& bytes, const int3* in, const uint8_t* keep, int3* out, int32_t* num_selected, int32_t f, cudaStream_t st)
{
    return cub::DeviceSelect::Flagged(tmp, bytes, in, keep, out, num_selected, f, st);
}
void cc_union(int32_t f, const int3* faces, int32_t* parent, cudaStream_t st) { k_cc_union<<<blocks(f), kThreads, 0, st>>>(f, faces, parent); }
void cc_flatten(int32_t nv, int32_t* parent, cudaStream_t st) { k_cc_flatten<<<blocks(nv), kThreads, 0, st>>>(nv, parent); }
void cc_count(int32_t f, const int3* faces, const int32_t* root, unsigned* count, unsigned* min_face, cudaStream_t st)
{
    k_cc_count<<<blocks(f), kThreads, 0, st>>>(f, faces, root, count, min_face);
}
void cc_best(int32_t nv, const unsigned* count, const unsigned* min_face, unsigned long long* best, cudaStream_t st)
{
    k_cc_best<<<blocks(nv), kThreads, 0, st>>>(nv, count, min_face, best);
}
void cc_keep(int32_t f, const int3* faces, const int32_t* root, const unsigned long long* best, uint8_t* keep, cudaStream_t st)
{
    k_cc_keep<<<blocks(f), kThreads, 0, st>>>(f, faces, root, best, keep);
}
void mark_used(int32_t f, const int3* faces, int32_t* used, cudaStream_t st) { k_mark_used<<<blocks(f), kThreads, 0, st>>>(f, faces, used); }
void compact_vertices(int32_t nv, const int32_t* used, const int32_t* new_id, const float* vpos, const uint8_t* vcol, float* vpos_out,
                      uint8_t* vcol_out, cudaStream_t st)
{
    k_compact_vertices<<<blocks(nv), kThreads, 0, st>>>(nv, used, new_id, vpos, vcol, vpos_out, vcol_out);
}
void remap_faces(int32_t f, const int32_t* new_id, int3* faces, cudaStream_t st) { k_remap_faces<<<blocks(f), kThreads, 0, st>>>(f, new_id, faces); }

} // namespace mesh
} // namespace i3d
