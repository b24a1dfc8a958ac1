// Intrinsic3D::refine on ONE resident H100 engine.  Reference control flow: src/refinement/intrinsic3d.cpp:206-409.
#include <nv/refinement/intrinsic3d.h>

#include <algorithm>
#include <cstring>
#include <iostream>
#include <sstream>

#include <nv/sdf/algorithms.h>

#include "../../include/i3d_c_api.h"

namespace nv
{
void Intrinsic3D::Config::load(const std::map<std::string, std::string>& s)
{
    auto num = [&](const char* k, double def) { auto it = s.find(k); if (it == s.end()) return def; std::istringstream is(it->second); double v = def; is >> v; return v; };
    num_grid_levels = static_cast<int>(num("num_grid_levels", num_grid_levels));
    thres_shell_factor = num("thin_shell_factor", thres_shell_factor);
    thres_shell_factor_final = num("thin_shell_factor_final", thres_shell_factor_final);
    clear_distant_voxels = num("clear_distant_voxels", clear_distant_voxels) != 0.0;
    num_rgbd_levels = static_cast<int>(num("num_rgbd_levels", num_rgbd_levels));
    occlusions_distance = static_cast<float>(num("occlusion_distance", occlusions_distance));
    num_observations = static_cast<size_t>(num("num_observations", static_cast<double>(num_observations)));
    subvolume_size_sh = static_cast<float>(num("subvolume_size_sh", subvolume_size_sh));
    sh_est_lambda_reg = num("subvolume_sh_lamda_reg", sh_est_lambda_reg);
}

void Intrinsic3D::Config::print() const
{
    std::cout << "Intrinsic3D config:" << std::endl;
    std::cout << "   num_grid_levels: " << num_grid_levels << std::endl << "   num_rgbd_levels: " << num_rgbd_levels << std::endl;
    std::cout << "   thres_shell_factor: " << thres_shell_factor << std::endl << "   thres_shell_factor_final: " << thres_shell_factor_final << std::endl;
    std::cout << "   clear_distant_voxels: " << clear_distant_voxels << std::endl << "   occlusions_distance: " << occlusions_distance << std::endl;
    std::cout << "   num_observations: " << num_observations << std::endl << "   subvolume_size_sh: " << subvolume_size_sh << std::endl;
    std::cout << "   sh_est_lambda_reg: " << sh_est_lambda_reg << std::endl;
}

Intrinsic3D::Intrinsic3D(Config cfg, Optimizer::Config opt_cfg, Optimizer::ImageFormationModel* image_model)
    : image_model_(image_model), opt_cfg_(opt_cfg), cfg_(cfg)
{
}

Intrinsic3D::~Intrinsic3D() { delete grid_; }

namespace
{
struct Flat
{
    std::vector<int32_t> xyz;
    std::vector<double> sdf0, sdf, alb;
    std::vector<float> weight;
    std::vector<uint8_t> rgb;
    void resize(size_t n) { xyz.resize(3 * n); sdf0.resize(n); sdf.resize(n); alb.resize(n); weight.resize(n); rgb.resize(3 * n); }
};

// host grid <- device grid (coordinates may have changed: prune / upsample)
bool pull_grid(I3DEngine* eng, SparseVoxelGrid<VoxelSBR>*& grid)
{
    const size_t n = static_cast<size_t>(i3d_num_voxels(eng));
    Flat f; f.resize(n);
    float vs = 0.0f;
    if (i3d_download_grid(eng, f.xyz.data(), f.sdf0.data(), f.sdf.data(), f.alb.data(), f.weight.data(), f.rgb.data(), &vs) != 0) return false;
    if (!grid || grid->voxelSize() != vs) { delete grid; grid = SparseVoxelGrid<VoxelSBR>::create(vs); }
    grid->clear();
    grid->reserve(n);
    for (size_t i = 0; i < n; ++i)
    {
        VoxelSBR v;
        v.sdf = f.sdf0[i]; v.sdf_refined = f.sdf[i]; v.albedo = f.alb[i]; v.weight = f.weight[i];
        v.color = Vec3b{f.rgb[3 * i], f.rgb[3 * i + 1], f.rgb[3 * i + 2]};
        grid->setVoxel(Vec3i{f.xyz[3 * i], f.xyz[3 * i + 1], f.xyz[3 * i + 2]}, v);
    }
    return true;
}
} // namespace

bool Intrinsic3D::refine(SparseVoxelGrid<Voxel>* grid_in)
{
    if (!grid_in) return false;
    if (cfg_.num_grid_levels <= 0 || cfg_.num_rgbd_levels <= 0) return false;
    if (!image_model_ || image_model_->poses.empty() || image_model_->rgbd_pyr.size() != image_model_->poses.size())
    {
        std::cerr << "Intrinsic3D::refine: no keyframe views" << std::endl;
        return false;
    }
    Optimizer::ImageFormationModel& im = *image_model_;
    const size_t F = im.poses.size();
    // Keyframes that carry only level 0 and its colour image: the engine builds the coarser levels itself from a device frame store
    // (i3d_upload_rgbd_frames / i3d_use_rgbd_level).  Pyramids that carry every level are uploaded level by level from the host.
    bool device_pyramid = cfg_.num_rgbd_levels > 1;
    for (size_t f = 0; f < F; ++f)
        device_pyramid = device_pyramid && im.rgbd_pyr[f].levels() == 1 && !im.rgbd_pyr[f].color(0).empty();
    for (size_t f = 0; f < F; ++f)
        if ((!device_pyramid && im.rgbd_pyr[f].levels() < cfg_.num_rgbd_levels) || im.rgbd_pyr[f].color(0).empty())
        {
            std::cerr << "Intrinsic3D::refine: frame " << f << " lacks pyramid levels or its colour image" << std::endl;
            return false;
        }
    std::cout << "Intrinsic3D ..." << std::endl;
    // fill initial grid on coarsest hierarchy level (SDFAlgorithms::convert)
    delete grid_;
    grid_ = SDFAlgorithms::convert(grid_in);
    if (!grid_ || grid_->empty()) return false;

    I3DEngine* eng = nullptr;
    if (i3d_engine_create(device_, &eng) != 0) { std::cerr << "Intrinsic3D::refine: " << i3d_last_error(nullptr) << std::endl; return false; }
    auto fail = [&](const char* what) { std::cerr << "Intrinsic3D::refine: " << what << ": " << i3d_last_error(eng) << std::endl; i3d_engine_destroy(eng); return false; };

    // ---- upload the grid once
    {
        const size_t n = grid_->numVoxels();
        Flat f; f.resize(n);
        size_t i = 0;
        for (auto it = grid_->begin(); it != grid_->end(); ++it, ++i)
        {
            const Vec3i& p = it->first; const VoxelSBR& v = it->second;
            f.xyz[3 * i] = p[0]; f.xyz[3 * i + 1] = p[1]; f.xyz[3 * i + 2] = p[2];
            f.sdf0[i] = v.sdf; f.sdf[i] = v.sdf_refined; f.alb[i] = v.albedo; f.weight[i] = v.weight;
            f.rgb[3 * i] = v.color[0]; f.rgb[3 * i + 1] = v.color[1]; f.rgb[3 * i + 2] = v.color[2];
        }
        if (i3d_upload_grid(eng, static_cast<int64_t>(n), f.xyz.data(), f.sdf0.data(), f.sdf.data(), f.alb.data(), f.weight.data(), f.rgb.data(), grid_->voxelSize()) != 0)
            return fail("upload grid");
    }
    float voxel_size = grid_->voxelSize();

    // frames of one pyramid level, packed; the luminance/depth planes go to the engine, the level-0 colour planes too
    std::vector<float> lum, depth;
    std::vector<uint8_t> color;
    int cur_level = -1;
    bool color_resident = false;
    if (device_pyramid)
    {
        const ImageF l0 = im.rgbd_pyr[0].intensity(0);
        const int W = l0.cols, H = l0.rows;
        const size_t px = static_cast<size_t>(W) * H;
        lum.resize(F * px); depth.resize(F * px); color.resize(F * px * 3);
        for (size_t f = 0; f < F; ++f)
        {
            const ImageF l = im.rgbd_pyr[f].intensity(0), d = im.rgbd_pyr[f].depth(0);
            const ImageBGR c = im.rgbd_pyr[f].color(0);
            if (l.rows != H || l.cols != W || d.rows != H || d.cols != W || c.rows != H || c.cols != W) return fail("keyframes of different sizes");
            std::memcpy(&lum[f * px], l.data, px * sizeof(float));
            std::memcpy(&depth[f * px], d.data, px * sizeof(float));
            std::memcpy(&color[f * px * 3], c.data, px * 3);
        }
        if (i3d_upload_rgbd_frames(eng, static_cast<int32_t>(F), W, H, color.data(), depth.data(), lum.data()) != 0) return fail("upload keyframes");
        std::vector<float>().swap(lum); std::vector<float>().swap(depth); std::vector<uint8_t>().swap(color);
    }
    auto upload_level = [&](int lvl, bool with_color) -> bool {
        if (device_pyramid)
        {
            // a level switch builds the level on the device; level 0 brings the colour planes along
            if (lvl != cur_level || (with_color && !color_resident))
            {
                if (i3d_use_rgbd_level(eng, lvl, nullptr, nullptr) != 0) return false;
                cur_level = lvl;
                color_resident = lvl == 0;
            }
            return !with_color || color_resident;
        }
        const ImageF l0 = im.rgbd_pyr[0].intensity(lvl);
        const int W = l0.cols, H = l0.rows;
        const size_t px = static_cast<size_t>(W) * H;
        if (lvl != cur_level)
        {
            lum.resize(F * px); depth.resize(F * px);
            for (size_t f = 0; f < F; ++f)
            {
                const ImageF l = im.rgbd_pyr[f].intensity(lvl), d = im.rgbd_pyr[f].depth(lvl);
                if (l.rows != H || l.cols != W || d.rows != H || d.cols != W) return false;
                std::memcpy(&lum[f * px], l.data, px * sizeof(float));
                std::memcpy(&depth[f * px], d.data, px * sizeof(float));
            }
            if (i3d_upload_frames(eng, static_cast<int32_t>(F), W, H, lum.data(), depth.data(), pyramidLevelToScale(lvl)) != 0) return false;
            cur_level = lvl;
            color_resident = false;          // a size change drops the colour planes on the device
        }
        if (with_color && !color_resident)
        {
            color.resize(F * px * 3);
            for (size_t f = 0; f < F; ++f)
            {
                const ImageBGR c = im.rgbd_pyr[f].color(lvl);
                if (c.rows != H || c.cols != W) return false;
                std::memcpy(&color[f * px * 3], c.data, px * 3);
            }
            if (i3d_upload_color_frames(eng, color.data()) != 0) return false;
            color_resident = true;
        }
        return true;
    };
    std::vector<double> poses(6 * F);
    for (size_t f = 0; f < F; ++f) for (int k = 0; k < 6; ++k) poses[6 * f + k] = im.poses[f][k];
    // Intrinsic3D::init: distortion starts at zero (intrinsic3d.cpp:160), initial recolouring on the level-0 frames
    im.distortion_coeffs = Vec5::Zero();
    if (!upload_level(0, true)) return fail("upload frames");
    if (i3d_set_camera(eng, poses.data(), im.intrinsics.data(), im.distortion_coeffs.data()) != 0) return fail("set camera");
    auto recolor = [&]() -> bool {
        if (!upload_level(0, true)) return false;
        return i3d_recompute_colors(eng, nullptr, cfg_.occlusions_distance, static_cast<int32_t>(cfg_.num_observations), nullptr, nullptr) == 0;
    };
    std::cout << "   initial SDF recolorization ..." << std::endl;
    if (!recolor()) return fail("initial recolorization");

    I3DParams P;
    i3d_default_params(&P);
    P.occlusion_distance = cfg_.occlusions_distance;
    P.num_observations = static_cast<int32_t>(cfg_.num_observations);
    P.lm_steps = opt_cfg_.lm_steps;
    P.use_er = opt_cfg_.lambda_r0 > 0.0 && opt_cfg_.lambda_r1 > 0.0;
    P.use_es = opt_cfg_.lambda_s0 > 0.0 && opt_cfg_.lambda_s1 > 0.0;
    P.use_ea = opt_cfg_.lambda_a > 0.0;
    P.fix_all_albedo = opt_cfg_.lambda_a < 0.0;
    P.fix_poses = opt_cfg_.fix_poses; P.fix_intrinsics = opt_cfg_.fix_intrinsics; P.fix_distortion = opt_cfg_.fix_distortion;
    I3DLightingParams LP;
    i3d_default_lighting_params(&LP);
    LP.subvolume_size = cfg_.subvolume_size_sh; LP.lambda_reg = cfg_.sh_est_lambda_reg; LP.weighted = 1;

    bool ok = true;
    bool emptied = false;              // the thin-shell pruning removed every voxel
    const int grid_lvl_coarsest = cfg_.num_grid_levels - 1;
    for (int grid_lvl = grid_lvl_coarsest; grid_lvl >= 0 && ok; --grid_lvl)
    {
        std::cout << "   refinement on level " << grid_lvl << std::endl << "      voxel size: " << voxel_size << std::endl << "      num voxels: " << i3d_num_voxels(eng) << std::endl;
        // ---- prepareGridLevel (intrinsic3d.cpp:296-316)
        double factor = cfg_.thres_shell_factor;
        if (cfg_.thres_shell_factor_final > 0.0)
            factor = computeVaryingLambda(grid_lvl_coarsest - grid_lvl, cfg_.num_grid_levels, cfg_.thres_shell_factor, cfg_.thres_shell_factor_final);
        const double thres_shell = factor * static_cast<double>(voxel_size);
        if (cfg_.clear_distant_voxels && !emptied)
        {
            int64_t m = 0;
            if (i3d_clear_voxels_outside_thin_shell(eng, thres_shell, &m) != 0) return fail("clear voxels outside thin shell");
            std::cout << "      num voxels (sparsified): " << m << std::endl;
            // nothing survives: the reference carries an empty grid through the remaining levels (every lighting estimate fails, the
            // level is skipped) and still returns true
            if (m == 0) emptied = true;
        }
        P.thres_shell = thres_shell; LP.thres_shell = thres_shell;
        const int rgbd_lvl_coarsest = cfg_.num_rgbd_levels - 1;
        for (int rgbd_lvl = rgbd_lvl_coarsest; rgbd_lvl >= 0; --rgbd_lvl)
        {
            if (rgbd_lvl > 0 && grid_lvl < grid_lvl_coarsest) continue;      // all pyramid levels only on the coarsest grid level
            std::cout << "   level " << grid_lvl << " (pyramid level " << rgbd_lvl << ") ..." << std::endl;
            if (emptied) { std::cerr << "   lighting estimation on level " << grid_lvl << " not successful!" << std::endl; break; }
            // ---- prepareRgbdLevel
            if (!upload_level(rgbd_lvl, false)) return fail("upload frames");
            // ---- lighting (intrinsic3d.cpp:253-268)
            I3DLightingInfo li;
            if (i3d_estimate_lighting(eng, &LP, &li) != 0) return fail("estimate lighting");
            if (!li.usable) { std::cerr << "   lighting estimation on level " << grid_lvl << " not successful!" << std::endl; break; }
            // ---- Optimizer::optimize (optimizer.cpp:119-171)
            for (int itr = 0; itr < opt_cfg_.iterations; ++itr)
            {
                P.lambda[0] = opt_cfg_.lambda_g;
                P.lambda[1] = computeVaryingLambda(itr, opt_cfg_.iterations, opt_cfg_.lambda_r0, opt_cfg_.lambda_r1);
                P.lambda[2] = computeVaryingLambda(itr, opt_cfg_.iterations, opt_cfg_.lambda_s0, opt_cfg_.lambda_s1);
                P.lambda[3] = opt_cfg_.lambda_a;
                I3DIterInfo info;
                if (i3d_gn_iteration(eng, &P, &info) != 0) { std::cerr << "   optimization failed! " << i3d_last_error(eng) << std::endl; break; }
            }
            // ---- finishRgbdLevel: recolouring with the refined camera model (intrinsic3d.cpp:347-378)
            if (!recolor()) return fail("recolorization");
            if (!callbacks_.empty())
            {
                if (!pull_grid(eng, grid_)) return fail("download grid");
                const RefinementInfo info{grid_lvl, cfg_.num_grid_levels, grid_, rgbd_lvl, cfg_.num_rgbd_levels};
                for (RefinementCallback* cb : callbacks_) cb->onSDFRefined(info);
            }
        }
        // ---- finishGridLevel
        if (grid_lvl > 0)
        {
            std::cout << "   upsampling grid for next level ..." << std::endl;
            int64_t m = 0;
            if (!emptied && i3d_upsample_grid(eng, &m) != 0) return fail("upsample");
            voxel_size = voxel_size * 0.5f;
        }
    }
    // ---- results back to the host structures
    if (emptied) { delete grid_; grid_ = SparseVoxelGrid<VoxelSBR>::create(voxel_size); }
    else if (!pull_grid(eng, grid_)) return fail("download grid");
    double intr[4], dist[5];
    if (i3d_download_state(eng, nullptr, nullptr, poses.data(), intr, dist) != 0) return fail("download camera");
    for (size_t f = 0; f < F; ++f) for (int k = 0; k < 6; ++k) im.poses[f][k] = poses[6 * f + k];
    for (int k = 0; k < 4; ++k) im.intrinsics[k] = intr[k];
    for (int k = 0; k < 5; ++k) im.distortion_coeffs[k] = dist[k];
    i3d_engine_destroy(eng);
    return ok;
}
} // namespace nv
