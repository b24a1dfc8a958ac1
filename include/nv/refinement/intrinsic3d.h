// nv/refinement/intrinsic3d.h — the refinement orchestrator with the reference's control flow
// (libintrinsic3d/include/nv/refinement/intrinsic3d.h:60-176, src/refinement/intrinsic3d.cpp:206-409), driving ONE resident
// H100 engine through the C-ABI for the whole coarse-to-fine schedule:
//
//   refine(grid):  convert -> init (initial recolouring) ->
//     for grid level (coarse -> fine):   prepareGridLevel   thin-shell threshold + i3d_clear_voxels_outside_thin_shell
//       for rgb-d pyramid level:         prepareRgbdLevel   i3d_upload_frames(level)
//                                        lighting           i3d_estimate_lighting
//                                        Optimizer          `iterations` x i3d_gn_iteration (lambda ramps as Optimizer::optimize)
//                                        finishRgbdLevel    i3d_recompute_colors on the level-0 frames; callbacks
//                                        finishGridLevel    i3d_upsample_grid
//   The grid, the camera parameters and the voxel colours stay on the device between the steps; the host copy is refreshed
//   when callbacks are registered and at the end.
//
// Difference from the reference's constructor: the keyframe views arrive prepared in an Optimizer::ImageFormationModel
// (poses, intrinsics, per-frame pyramids with colour) instead of being pulled from Sensor / KeyframeSelection — frame IO, keyframe
// selection and pyramid construction are image preparation outside the path (SURVEY.md §8, out of scope).
#pragma once
#include <map>
#include <string>
#include <vector>

#include <nv/refinement/optimizer.h>
#include <nv/sparse_voxel_grid.h>

namespace nv
{
class Intrinsic3D
{
public:
    // field names, ORDER and defaults of the reference's Config (intrinsic3d.h:71-90); keys of data/intrinsic3d.yml in load()
    struct Config
    {
        // sdf grid
        int num_grid_levels = 3;
        double thres_shell_factor = 2.0;           // thin shell, in voxel sizes, ramped over the grid levels
        double thres_shell_factor_final = 1.0;
        bool clear_distant_voxels = true;
        // rgbd frame sampling
        int num_rgbd_levels = 3;
        float occlusions_distance = 0.02f;         // observation visibility
        size_t num_observations = 5;               // best observations per voxel (0 = all)
        // svsh estimation
        float subvolume_size_sh = 0.2f;
        double sh_est_lambda_reg = 10.0;
        void load(const std::map<std::string, std::string>& settings);
        void print() const;
    };
    // what a RefinementCallback receives after every (grid level, pyramid level)
    struct RefinementInfo { int grid_level, num_grid_levels; SparseVoxelGrid<VoxelSBR>* grid; int pyramid_level, num_pyramid_levels; };
    class RefinementCallback
    {
    public:
        virtual void onSDFRefined(const RefinementInfo& info) = 0;
        virtual ~RefinementCallback() {}
    };

    Intrinsic3D(Config cfg, Optimizer::Config opt_cfg, Optimizer::ImageFormationModel* image_model);
    ~Intrinsic3D();

    bool refine(SparseVoxelGrid<Voxel>* grid);
    void addRefinementCallback(RefinementCallback* cb) { callbacks_.push_back(cb); }
    const Config& config() const { return cfg_; }
    // the refined grid of the last refine() (the reference hands it out through the callbacks only and deletes it at the end;
    // here it stays alive until the next refine() / destruction)
    SparseVoxelGrid<VoxelSBR>* refinedGrid() { return grid_; }
    void setDevice(int cuda_device) { device_ = cuda_device; }

private:
    std::vector<RefinementCallback*> callbacks_;
    Optimizer::ImageFormationModel* image_model_;
    SparseVoxelGrid<VoxelSBR>* grid_ = nullptr;
    Optimizer::Config opt_cfg_;
    Config cfg_;
    int device_ = 0;
};
} // namespace nv
