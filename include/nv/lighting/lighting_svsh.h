// nv/lighting/lighting_svsh.h — spatially-varying SH lighting with the reference's call surface (constructor arguments, estimate(),
// computeVoxelShCoeffs(), interpolate(), shCoeffs(), subvolumes(); libintrinsic3d/include/nv/lighting/lighting_svsh.h:47-70), computed by
// the H100 engine (i3d_estimate_lighting, include/i3d_c_api.h) instead of Ceres.
//
//   LightingSVSH lighting(grid, subvolume_size, lambda_reg, thres_shell, weighted);
//   if (!lighting.estimate()) ...                          // src/refinement/intrinsic3d.cpp:255-262
//   lighting.computeVoxelShCoeffs(data.voxel_sh_coeffs);    // :264
//
// estimate() runs the subvolume generation, the joint SH solve AND the per-voxel blend on the device in one call and keeps the
// results on the host; computeVoxelShCoeffs() hands out the already computed vectors (empty VecXd for the voxels the reference skips:
// invalid or outside the thin shell).
#pragma once
#include <cstdint>
#include <vector>

#include <nv/lighting/subvolumes.h>
#include <nv/mat.h>
#include <nv/sparse_voxel_grid.h>

namespace nv
{
class LightingSVSH
{
public:
    LightingSVSH(const SparseVoxelGrid<VoxelSBR>* grid, float subvolume_size, double lambda_reg, double thres_shell = 0.0, bool weighted = false);
    ~LightingSVSH();

    // the solve + the per-voxel blend (one engine call); false exactly when the reference's estimate() is
    bool estimate();
    bool computeVoxelShCoeffs(std::vector<VecXd>& voxel_coeffs) const;
    bool interpolate(const Vec3i& v_pos, VecXd& sh_coeffs) const;
    std::vector<VecXd> shCoeffs() const { return result_.subvolume_sh; }
    const Subvolumes& subvolumes() const { return result_.subvolumes; }

    // not in the reference: device choice and the ceres::Solver::Summary equivalents of the last estimate()
    void setDevice(int cuda_device) { device_ = cuda_device; }
    int iterations() const { return result_.iterations; }
    double initialCost() const { return result_.cost_initial; }
    double finalCost() const { return result_.cost_final; }

private:
    struct Inputs
    {
        const SparseVoxelGrid<VoxelSBR>* grid;
        float subvolume_size;
        double lambda_reg, thres_shell;
        bool weighted;
    };
    struct Result
    {
        explicit Result(float size) : subvolumes(size) {}
        Subvolumes subvolumes;
        std::vector<VecXd> subvolume_sh;      // [S] 9-vectors
        std::vector<double> voxel_sh;         // [n][9] blend computed on the device
        std::vector<uint8_t> voxel_has_sh;    // [n]
        int iterations = 0;
        double cost_initial = 0.0, cost_final = 0.0;
    };
    Inputs in_;
    Result result_;
    int device_ = 0;
};
} // namespace nv
