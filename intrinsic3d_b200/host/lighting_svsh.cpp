// LightingSVSH / Subvolumes on the H100 engine.  Reference: src/lighting/lighting_svsh.cpp:54-346, src/lighting/subvolumes.cpp.
#include <nv/lighting/lighting_svsh.h>

#include <iostream>

#include "../../include/i3d_c_api.h"

namespace nv
{
VecXd Subvolumes::interpolate(const std::vector<VecXd>& values, const Vec3f& pt, bool linear) const
{
    VecXd avg(values.empty() ? 0 : values[0].size(), 0.0);
    if (!linear)
    {
        const int s = pointToSubvolume(pt);
        if (s >= 0) avg = values[static_cast<size_t>(s)];
        return avg;
    }
    // math::interpolationWeights + math::average (src/math.cpp:74-128): float weights, missing cubes dropped, renormalised
    const Vec3f pos = pointToIndexCoord(pt);
    int v0[3]; float t[3];
    for (int d = 0; d < 3; ++d) { v0[d] = static_cast<int>(std::floor(pos[d])); t[d] = pos[d] - static_cast<float>(v0[d]); }
    static const int corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {0, 0, 1}, {1, 1, 0}, {0, 1, 1}, {1, 0, 1}, {1, 1, 1}};
    float sum_w = 0.0f;
    for (int c = 0; c < 8; ++c)
    {
        const float w = (corner[c][0] ? t[0] : 1.0f - t[0]) * (corner[c][1] ? t[1] : 1.0f - t[1]) * (corner[c][2] ? t[2] : 1.0f - t[2]);
        const int s = indexToSubvolume(Vec3i{v0[0] + corner[c][0], v0[1] + corner[c][1], v0[2] + corner[c][2]});
        if (s < 0 || w == 0.0f) continue;
        const VecXd& val = values[static_cast<size_t>(s)];
        for (size_t k = 0; k < avg.size(); ++k) avg[k] = (sum_w == 0.0f) ? static_cast<double>(w) * val[k] : avg[k] + static_cast<double>(w) * val[k];
        sum_w += w;
    }
    if (sum_w != 0.0f) for (double& a : avg) a *= static_cast<double>(1.0f / sum_w);
    return avg;
}

LightingSVSH::LightingSVSH(const SparseVoxelGrid<VoxelSBR>* grid, float subvolume_size, double lambda_reg, double thres_shell, bool weighted)
    : in_{grid, subvolume_size, lambda_reg, thres_shell, weighted}, result_(subvolume_size)
{
}

LightingSVSH::~LightingSVSH() {}

bool LightingSVSH::estimate()
{
    result_ = Result(in_.subvolume_size);
    const SparseVoxelGrid<VoxelSBR>* grid = in_.grid;
    if (!grid || grid->empty() || in_.thres_shell <= 0.0) return false;          // lighting_svsh.cpp:170-171
    const size_t n = grid->numVoxels();
    std::vector<int32_t> xyz(3 * n);
    std::vector<double> sdf0(n), sdf(n), alb(n);
    std::vector<float> weight(n);
    std::vector<uint8_t> rgb(3 * n);
    size_t i = 0;
    for (auto it = grid->begin(); it != grid->end(); ++it, ++i)
    {
        const Vec3i& p = it->first; const VoxelSBR& v = it->second;
        xyz[3 * i] = p[0]; xyz[3 * i + 1] = p[1]; xyz[3 * i + 2] = p[2];
        sdf0[i] = v.sdf; sdf[i] = v.sdf_refined; alb[i] = v.albedo; weight[i] = v.weight;
        rgb[3 * i] = v.color[0]; rgb[3 * i + 1] = v.color[1]; rgb[3 * i + 2] = v.color[2];
    }
    I3DEngine* eng = nullptr;
    if (i3d_engine_create(device_, &eng) != 0) { std::cerr << "LightingSVSH::estimate: " << i3d_last_error(nullptr) << std::endl; return false; }
    auto fail = [&](const char* what) { std::cerr << "LightingSVSH::estimate: " << what << ": " << i3d_last_error(eng) << std::endl; i3d_engine_destroy(eng); return false; };
    if (i3d_upload_grid(eng, static_cast<int64_t>(n), xyz.data(), sdf0.data(), sdf.data(), alb.data(), weight.data(), rgb.data(), grid->voxelSize()) != 0)
        return fail("upload grid");
    I3DLightingParams P;
    i3d_default_lighting_params(&P);
    P.subvolume_size = in_.subvolume_size; P.lambda_reg = in_.lambda_reg; P.thres_shell = in_.thres_shell; P.weighted = in_.weighted ? 1 : 0;
    I3DLightingInfo info;
    std::cout << "Estimating local spherical harmonics (joint estimation over all subvolumes) ..." << std::endl;
    if (i3d_estimate_lighting(eng, &P, &info) != 0) return fail("estimate");
    std::cout << "number of generated SH subvolumes: " << info.num_subvolumes << "; " << info.num_data_rows << " voxel residuals, "
              << info.num_reg_pairs << " regularizer residuals; cost " << info.cost_initial << " -> " << info.cost_final << " in "
              << info.lm_iterations << " iterations" << std::endl;
    result_.iterations = info.lm_iterations; result_.cost_initial = info.cost_initial; result_.cost_final = info.cost_final;
    if (!info.usable) { i3d_engine_destroy(eng); return false; }
    const size_t S = static_cast<size_t>(info.num_subvolumes);
    std::vector<int32_t> index3(3 * S);
    std::vector<double> sh(9 * S);
    result_.voxel_sh.resize(9 * n); result_.voxel_has_sh.resize(n);
    if (i3d_download_lighting(eng, index3.data(), sh.data()) != 0) return fail("download lighting");
    if (i3d_download_voxel_sh(eng, result_.voxel_sh.data(), result_.voxel_has_sh.data()) != 0) return fail("download voxel sh");
    i3d_engine_destroy(eng);
    result_.subvolumes.assign(grid->voxelSize(), index3);
    result_.subvolume_sh.resize(S);
    for (size_t s = 0; s < S; ++s) result_.subvolume_sh[s].assign(sh.begin() + 9 * s, sh.begin() + 9 * s + 9);
    return true;
}

bool LightingSVSH::interpolate(const Vec3i& v_pos, VecXd& sh_coeffs) const
{
    if (!in_.grid || !in_.grid->valid(v_pos)) return false;
    const float vs = in_.grid->voxelSize();
    const Vec3f v_coord{static_cast<float>(v_pos[0]) * vs, static_cast<float>(v_pos[1]) * vs, static_cast<float>(v_pos[2]) * vs};   // voxelToWorld
    sh_coeffs = result_.subvolumes.interpolate(result_.subvolume_sh, v_coord, true);
    return true;
}

bool LightingSVSH::computeVoxelShCoeffs(std::vector<VecXd>& voxel_coeffs) const
{
    if (!in_.grid) return false;
    const size_t n = in_.grid->numVoxels();
    voxel_coeffs.clear();
    voxel_coeffs.resize(n, VecXd());
    if (result_.voxel_has_sh.size() != n) return result_.subvolume_sh.empty();      // estimate() not run on this grid
    for (size_t i = 0; i < n; ++i)
        if (result_.voxel_has_sh[i]) voxel_coeffs[i].assign(result_.voxel_sh.begin() + 9 * i, result_.voxel_sh.begin() + 9 * i + 9);
    return true;
}
} // namespace nv
