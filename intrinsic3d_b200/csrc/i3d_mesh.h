/*
 * i3d_mesh.h — host interface of the surface-extraction kernels (i3d_mesh.cuh, compiled in i3d_mesh.cu).  The kernels live in a
 * device module of their own, so the engine's module holds exactly the kernels of the refinement path; the engine (i3d_engine.cu)
 * owns the buffers and the stage order and calls these wrappers on its stream.  The CUB wrappers follow CUB's two-call convention:
 * with tmp == nullptr they only set `bytes`.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "i3d_grid.cuh"

namespace i3d
{

struct MeshGrid
{
    int64_t n;
    const int32_t* x; const int32_t* y; const int32_t* z;
    const double* sdf;              // sdf0 or the refined sdf
    const float* weight;
    const uchar4* rgb;
    const int32_t* nbr;             // [12][n]
    const unsigned long long* keys; const int32_t* vals; uint64_t mask;    // device hash of the grid, for the (1,1,1) corner
    float voxel_size;
};

// Corner buffers of the raw triangle soup, corner index = 3 * face + k: position, colour and the position's sort key (float bits
// with the sign of zero canonicalised: -0.0 and +0.0 compare equal, as in merge's std::map).
struct MeshCorners
{
    float* pos;                    // [3M]
    uint8_t* col;                  // [3M]
    uint32_t* key_lo;              // z bits
    unsigned long long* key_hi;    // x bits << 32 | y bits
};

namespace mesh
{
// 0. the per-voxel colours of a colour mode (i3d_vis.cuh; mode 1 .. I3D_MESH_COLOR_COUNT - 1) into out [n]; g.sdf is the sdf the mesh is
// cut from, sg / sub_sh [S][9] the subvolumes and subvolume SH of the last lighting estimate (read by the shading modes only)
void colorize(const GridView& g, const SubvolGrid& sg, const double* sub_sh, int S, int mode, uchar4* out, cudaStream_t st);
// 1. cube cases, triangle counts, used-cube count; face offsets (int64 exclusive scan of the counts)
void classify(const MeshGrid& g, uint8_t* cube_case, int32_t* tri_count, unsigned long long* num_cubes, cudaStream_t st);
cudaError_t face_offsets(void* tmp, size_t& bytes, const int32_t* tri_count, int64_t* face_off, int n, cudaStream_t st);
// 2. the triangle soup
void emit(const MeshGrid& g, const uint8_t* cube_case, const int32_t* tri_count, const int64_t* face_off, const MeshCorners& out, cudaStream_t st);
// 3. welding
void iota(int32_t m, int32_t* out, cudaStream_t st);
cudaError_t sort_z(void* tmp, size_t& bytes, const uint32_t* key_lo, uint32_t* key_lo_sorted, const int32_t* perm_in, int32_t* perm_out, int32_t m,
                   cudaStream_t st);
void gather_key_hi(int32_t m, const int32_t* perm, const unsigned long long* key_hi, unsigned long long* out, cudaStream_t st);
cudaError_t sort_xy(void* tmp, size_t& bytes, const unsigned long long* key_hi, unsigned long long* key_hi_sorted, const int32_t* perm_in,
                    int32_t* perm_out, int32_t m, cudaStream_t st);
void weld_heads(int32_t m, const int32_t* perm, const unsigned long long* hi_sorted, const uint32_t* key_lo, int32_t* is_first, int32_t* head_pos,
                cudaStream_t st);
cudaError_t exclusive_sum(void* tmp, size_t& bytes, const int32_t* in, int32_t* out, int32_t m, cudaStream_t st);
cudaError_t inclusive_max(void* tmp, size_t& bytes, const int32_t* in, int32_t* out, int32_t m, cudaStream_t st);
void weld_assign(int32_t m, const int32_t* perm, const int32_t* seg_head, const int32_t* first_id, const float* cpos, const uint8_t* ccol,
                 int32_t* corner_vid, float* vpos, uint8_t* vcol, cudaStream_t st);
// 4. degenerate faces; order-keeping selection of flagged faces
void face_clean(int32_t f, const int3* faces, const float* vpos, uint8_t* keep, cudaStream_t st);
cudaError_t select_faces(void* tmp, size_t& bytes, const int3* in, const uint8_t* keep, int3* out, int32_t* num_selected, int32_t f, cudaStream_t st);
// 5. largest component and the vertices it uses
void cc_union(int32_t f, const int3* faces, int32_t* parent, cudaStream_t st);
void cc_flatten(int32_t nv, int32_t* parent, cudaStream_t st);
void cc_count(int32_t f, const int3* faces, const int32_t* root, unsigned* count, unsigned* min_face, cudaStream_t st);
void cc_best(int32_t nv, const unsigned* count, const unsigned* min_face, unsigned long long* best, cudaStream_t st);
void cc_keep(int32_t f, const int3* faces, const int32_t* root, const unsigned long long* best, uint8_t* keep, cudaStream_t st);
void mark_used(int32_t f, const int3* faces, int32_t* used, cudaStream_t st);
void compact_vertices(int32_t nv, const int32_t* used, const int32_t* new_id, const float* vpos, const uint8_t* vcol, float* vpos_out,
                      uint8_t* vcol_out, cudaStream_t st);
void remap_faces(int32_t f, const int32_t* new_id, int3* faces, cudaStream_t st);
} // namespace mesh

} // namespace i3d
