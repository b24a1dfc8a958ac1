// SDFColorization::add / compute on the H100 engine.  Reference: src/sdf/colorization.cpp:113-189.
#include <nv/sdf/colorization.h>

#include <cstring>
#include <iostream>

#include "../../include/i3d_c_api.h"

namespace nv
{
bool SDFColorization::add(int id, const ImageF& depth, const ImageBGR& color, const Mat4f& pose_world_to_cam)
{
    if (!grid_ || grid_->empty()) return false;
    if (depth.rows != color.rows || depth.cols != color.cols)
    {
        std::cerr << "color and depth image sizes do not match!" << std::endl;
        return false;
    }
    if (!views_.empty() && (views_[0].depth.rows != depth.rows || views_[0].depth.cols != depth.cols))
    {
        std::cerr << "SDFColorization::add: all views must have the same size" << std::endl;
        return false;
    }
    views_.push_back(View{id, depth, color, pose_world_to_cam});
    return true;
}

bool SDFColorization::compute()
{
    if (!grid_ || grid_->empty() || views_.empty()) return false;
    const size_t n = grid_->numVoxels();
    const size_t F = views_.size();
    const int W = views_[0].depth.cols, H = views_[0].depth.rows;
    const size_t px = static_cast<size_t>(W) * H;
    std::vector<int32_t> xyz(3 * n);
    std::vector<double> sdf0(n), sdf(n), alb(n);
    std::vector<float> weight(n);
    std::vector<uint8_t> rgb(3 * n);
    size_t i = 0;
    for (auto it = grid_->begin(); it != grid_->end(); ++it, ++i)
    {
        const Vec3i& p = it->first; const VoxelSBR& v = it->second;
        xyz[3 * i] = p[0]; xyz[3 * i + 1] = p[1]; xyz[3 * i + 2] = p[2];
        sdf0[i] = v.sdf; sdf[i] = v.sdf_refined; alb[i] = v.albedo; weight[i] = v.weight;
        rgb[3 * i] = v.color[0]; rgb[3 * i + 1] = v.color[1]; rgb[3 * i + 2] = v.color[2];
    }
    std::vector<float> depth(F * px), rt(12 * F);
    std::vector<uint8_t> color(F * px * 3);
    std::vector<double> poses(6 * F, 0.0);
    for (size_t f = 0; f < F; ++f)
    {
        std::memcpy(&depth[f * px], views_[f].depth.data, px * sizeof(float));
        std::memcpy(&color[f * px * 3], views_[f].color.data, px * 3);
        const Mat4f& P = views_[f].pose;
        for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) rt[12 * f + 3 * r + c] = P(r, c); rt[12 * f + 9 + r] = P(r, 3); }
    }
    I3DEngine* eng = nullptr;
    if (i3d_engine_create(device_, &eng) != 0) { std::cerr << "SDFColorization::compute: " << i3d_last_error(nullptr) << std::endl; return false; }
    auto fail = [&](const char* what) { std::cerr << "SDFColorization::compute: " << what << ": " << i3d_last_error(eng) << std::endl; i3d_engine_destroy(eng); return false; };
    if (i3d_upload_grid(eng, static_cast<int64_t>(n), xyz.data(), sdf0.data(), sdf.data(), alb.data(), weight.data(), rgb.data(), grid_->voxelSize()) != 0)
        return fail("upload grid");
    // the luminance plane is not read by the recolouring pass: the depth plane stands in for it
    if (i3d_upload_frames(eng, static_cast<int32_t>(F), W, H, depth.data(), depth.data(), 1.0) != 0) return fail("upload frames");
    if (i3d_upload_color_frames(eng, color.data()) != 0) return fail("upload colour frames");
    if (i3d_set_camera(eng, poses.data(), intrinsics_.data(), dist_.data()) != 0) return fail("set camera");
    int64_t n_col = 0, n_obs = 0;
    if (i3d_recompute_colors(eng, rt.data(), cfg_.max_occlusion_distance, static_cast<int32_t>(cfg_.max_num_observations), &n_col, &n_obs) != 0)
        return fail("recompute colours");
    if (i3d_download_colors(eng, rgb.data()) != 0) return fail("download colours");
    i3d_engine_destroy(eng);
    i = 0;
    for (auto it = grid_->begin(); it != grid_->end(); ++it, ++i) it->second.color = Vec3b{rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]};
    views_.clear();
    return true;
}
} // namespace nv
