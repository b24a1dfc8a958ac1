// nv/refinement/optimizer.h — Optimizer with the reference's API surface (include/nv/refinement/optimizer.h:59-141), driving the
// H100 engine through the C-ABI (include/i3d_c_api.h) instead of Ceres.
//
// optimize() mutates, in place and like the reference: grid voxels' sdf_refined / albedo, image_formation.poses /
// intrinsics / distortion_coeffs.  Returns false only if the grid is null or iterations < 1 (optimizer.cpp:113-114) or if the
// engine reports an error (message on std::cerr).
#pragma once
#include <map>
#include <string>
#include <unordered_set>
#include <vector>

#include <nv/mat.h>
#include <nv/refinement/nls_solver.h>
#include <nv/refinement/shading_cost.h>
#include <nv/rgbd/pyramid.h>
#include <nv/sdf/colorization.h>
#include <nv/sparse_voxel_grid.h>

namespace nv
{
class Optimizer
{
public:
    // field names, ORDER and defaults of the reference's Optimizer::Config (optimizer.h:67-88): aggregate initialisation written
    // against the reference keeps working
    struct Config
    {
        int iterations = 10;          // outer GN iterations
        int lm_steps = 50;            // ceres max_num_iterations
        double lambda_g = 0.2;        // shading-gradient data term
        double lambda_r0 = 20.0;      // volumetric regulariser, ramp start
        double lambda_r1 = 160.0;     //                         ramp end
        double lambda_s0 = 10.0;      // surface stabiliser, ramp start
        double lambda_s1 = 120.0;     //                     ramp end
        double lambda_a = 0.1;        // albedo regulariser (< 0: all albedos fixed)
        bool fix_poses = false;
        bool fix_intrinsics = false;
        bool fix_distortion = false;
        // flat key -> value settings with the key names of data/intrinsic3d.yml (the reference reads them through
        // nv::Settings / cv::FileStorage, src/refinement/optimizer.cpp:52-72: OUT-OF-SCOPE types, see INTEGRATION.md); missing keys
        // keep the defaults above
        void load(const std::map<std::string, std::string>& settings);
        void print() const;
    };
    // what optimize() reads besides the camera model (reference: optimizer.h:91-100, same order); the grid is NOT owned
    struct Data
    {
        SparseVoxelGrid<VoxelSBR>* grid = nullptr;
        double thres_shell = 0.0;
        int grid_level = 0;
        int rgbd_level = 0;
        std::vector<VecXd> voxel_sh_coeffs;                           // per voxel, indexed by the grid's iteration order
        std::vector<ShadingCostData> shading_cost_data;               // per frame
        std::unordered_set<Vec3i, std::hash<Vec3i>> voxels_added;    // scratch of the reference's serial loop; unused here
    };
    // camera model + keyframes, mutated in place (reference: optimizer.h:107-115, same order)
    struct ImageFormationModel
    {
        Vec4 intrinsics = Vec4::Zero();          // fx, fy, cx, cy at full resolution
        Vec5 distortion_coeffs = Vec5::Zero();   // k1, k2, k3, p1, p2
        std::vector<int> frame_ids;
        std::vector<Vec6> poses;                 // world -> camera: angle-axis, translation
        std::vector<Pyramid> rgbd_pyr;           // one per pose
    };

    explicit Optimizer(Config cfg);
    ~Optimizer();
    const Config& config() const;
    bool optimize(SDFColorization& colorization, Data& data, ImageFormationModel& image_formation);

    // per outer iteration diagnostics of the last optimize() call (NLSSolver::ProblemInfo / SolverInfo)
    const std::vector<NLSSolver::ProblemInfo>& problemInfo() const { return problem_info_; }
    const std::vector<NLSSolver::SolverInfo>& solverInfo() const { return solver_info_; }
    void setDevice(int cuda_device) { device_ = cuda_device; }

private:
    Config cfg_;
    int device_ = 0;
    std::vector<NLSSolver::ProblemInfo> problem_info_;
    std::vector<NLSSolver::SolverInfo> solver_info_;
};
} // namespace nv
