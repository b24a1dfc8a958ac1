// SDFAlgorithms::clearVoxelsOutsideThinShell / upsample on the H100 engine.  Reference: src/sdf/algorithms.cpp:118-235, 368-458.
#include <nv/sdf/algorithms.h>

#include <iostream>

#include "../../include/i3d_c_api.h"

namespace nv
{
namespace SDFAlgorithms
{
namespace
{
int g_device = 0;

struct Flat
{
    std::vector<int32_t> xyz;
    std::vector<double> sdf0, sdf, alb;
    std::vector<float> weight;
    std::vector<uint8_t> rgb;
    void resize(size_t n) { xyz.resize(3 * n); sdf0.resize(n); sdf.resize(n); alb.resize(n); weight.resize(n); rgb.resize(3 * n); }
};

I3DEngine* upload(const SparseVoxelGrid<VoxelSBR>* grid, const char* who)
{
    const size_t n = grid->numVoxels();
    Flat f; f.resize(n);
    size_t i = 0;
    for (auto it = grid->begin(); it != grid->end(); ++it, ++i)
    {
        const Vec3i& p = it->first; const VoxelSBR& v = it->second;
        f.xyz[3 * i] = p[0]; f.xyz[3 * i + 1] = p[1]; f.xyz[3 * i + 2] = p[2];
        f.sdf0[i] = v.sdf; f.sdf[i] = v.sdf_refined; f.alb[i] = v.albedo; f.weight[i] = v.weight;
        f.rgb[3 * i] = v.color[0]; f.rgb[3 * i + 1] = v.color[1]; f.rgb[3 * i + 2] = v.color[2];
    }
    I3DEngine* eng = nullptr;
    if (i3d_engine_create(g_device, &eng) != 0) { std::cerr << who << ": " << i3d_last_error(nullptr) << std::endl; return nullptr; }
    if (i3d_upload_grid(eng, static_cast<int64_t>(n), f.xyz.data(), f.sdf0.data(), f.sdf.data(), f.alb.data(), f.weight.data(), f.rgb.data(), grid->voxelSize()) != 0)
    {
        std::cerr << who << ": upload grid: " << i3d_last_error(eng) << std::endl;
        i3d_engine_destroy(eng);
        return nullptr;
    }
    return eng;
}

bool download(I3DEngine* eng, SparseVoxelGrid<VoxelSBR>* out, const char* who)
{
    const size_t n = static_cast<size_t>(i3d_num_voxels(eng));
    Flat f; f.resize(n);
    float vs = 0.0f;
    if (i3d_download_grid(eng, f.xyz.data(), f.sdf0.data(), f.sdf.data(), f.alb.data(), f.weight.data(), f.rgb.data(), &vs) != 0)
    {
        std::cerr << who << ": download grid: " << i3d_last_error(eng) << std::endl;
        return false;
    }
    out->clear();
    out->reserve(n);
    for (size_t i = 0; i < n; ++i)
    {
        VoxelSBR v;
        v.sdf = f.sdf0[i]; v.sdf_refined = f.sdf[i]; v.albedo = f.alb[i]; v.weight = f.weight[i];
        v.color = Vec3b{f.rgb[3 * i], f.rgb[3 * i + 1], f.rgb[3 * i + 2]};
        out->setVoxel(Vec3i{f.xyz[3 * i], f.xyz[3 * i + 1], f.xyz[3 * i + 2]}, v);
    }
    return true;
}
} // namespace

void setDevice(int cuda_device) { g_device = cuda_device; }

std::vector<Vec3i> collectRingNeighborhood(const Vec3i& p)
{
    return {Vec3i{p[0] + 1, p[1], p[2]}, Vec3i{p[0] - 1, p[1], p[2]}, Vec3i{p[0], p[1] + 1, p[2]},
            Vec3i{p[0], p[1] - 1, p[2]}, Vec3i{p[0], p[1], p[2] + 1}, Vec3i{p[0], p[1], p[2] - 1}};
}

SparseVoxelGrid<VoxelSBR>* convert(SparseVoxelGrid<Voxel>* grid)
{
    if (!grid) return nullptr;
    SparseVoxelGrid<VoxelSBR>* out = SparseVoxelGrid<VoxelSBR>::create(grid->voxelSize(), grid->depthMin(), grid->depthMax());
    out->reserve(grid->numVoxels());
    for (auto it = grid->begin(); it != grid->end(); ++it)
    {
        const Voxel& v = it->second;
        if (!(v.weight > 0.0f)) continue;                   // clearInvalidVoxels (algorithms.cpp:341-365)
        VoxelSBR s;
        s.sdf = static_cast<double>(v.sdf); s.color = v.color; s.weight = v.weight; s.sdf_refined = static_cast<double>(v.sdf);
        out->setVoxel(it->first, s);
    }
    return out;
}

void clearVoxelsOutsideThinShell(SparseVoxelGrid<VoxelSBR>* grid, double thres_shell)
{
    if (!grid || grid->empty()) return;
    I3DEngine* eng = upload(grid, "clearVoxelsOutsideThinShell");
    if (!eng) return;
    int64_t m = 0;
    if (i3d_clear_voxels_outside_thin_shell(eng, thres_shell, &m) != 0)
        std::cerr << "clearVoxelsOutsideThinShell: " << i3d_last_error(eng) << std::endl;       // grid left untouched
    else
        download(eng, grid, "clearVoxelsOutsideThinShell");
    i3d_engine_destroy(eng);
}

SparseVoxelGrid<VoxelSBR>* upsample(const SparseVoxelGrid<VoxelSBR>* grid)
{
    if (!grid) return nullptr;
    SparseVoxelGrid<VoxelSBR>* up = SparseVoxelGrid<VoxelSBR>::create(grid->voxelSize() * 0.5f);
    if (!up || grid->empty()) return up;
    I3DEngine* eng = upload(grid, "upsample");
    if (!eng) { delete up; return nullptr; }
    int64_t m = 0;
    bool ok = i3d_upsample_grid(eng, &m) == 0;
    if (!ok) std::cerr << "upsample: " << i3d_last_error(eng) << std::endl;
    ok = ok && download(eng, up, "upsample");
    i3d_engine_destroy(eng);
    if (!ok) { delete up; return nullptr; }
    return up;
}
} // namespace SDFAlgorithms
} // namespace nv
