// Optimizer::optimize on the H100 engine.  Reference: src/refinement/optimizer.cpp:109-173 (outer loop), :285-361 (fixing).
// Per call: flatten the hash grid in its iteration order, upload grid / frames / camera / SH once, run `iterations`
// outer Gauss-Newton iterations on the device (state stays resident), write the refined parameters back in place.
#include <nv/refinement/optimizer.h>

#include <cstdlib>
#include <iostream>
#include <sstream>

#include "../../include/i3d_c_api.h"

namespace nv
{
void Optimizer::Config::load(const std::map<std::string, std::string>& s)
{
    auto num = [&](const char* k, double def) { auto it = s.find(k); if (it == s.end()) return def; std::istringstream is(it->second); double v = def; is >> v; return v; };
    iterations = static_cast<int>(num("iterations", iterations));
    lm_steps = static_cast<int>(num("lm_steps", lm_steps));
    lambda_g = num("lambda_g", lambda_g);
    lambda_r0 = num("lambda_r0", lambda_r0); lambda_r1 = num("lambda_r1", lambda_r1);
    lambda_s0 = num("lambda_s0", lambda_s0); lambda_s1 = num("lambda_s1", lambda_s1);
    lambda_a = num("lambda_a", lambda_a);
    fix_poses = num("fix_poses", fix_poses) != 0.0; fix_intrinsics = num("fix_intrinsics", fix_intrinsics) != 0.0; fix_distortion = num("fix_distortion", fix_distortion) != 0.0;
}

void Optimizer::Config::print() const
{
    std::cout << "Optimizer config: iterations " << iterations << ", lm_steps " << lm_steps << ", lambda_g " << lambda_g << ", lambda_r " << lambda_r0 << "->"
              << lambda_r1 << ", lambda_s " << lambda_s0 << "->" << lambda_s1 << ", lambda_a " << lambda_a << ", fix poses/intrinsics/distortion " << fix_poses
              << "/" << fix_intrinsics << "/" << fix_distortion << std::endl;
}

Optimizer::Optimizer(Config cfg) : cfg_(cfg) {}
Optimizer::~Optimizer() {}
const Optimizer::Config& Optimizer::config() const { return cfg_; }

bool Optimizer::optimize(SDFColorization& colorization, Data& data, ImageFormationModel& im)
{
    if (!data.grid || cfg_.iterations < 1) return false;
    SparseVoxelGrid<VoxelSBR>* grid = data.grid;
    const size_t n = grid->numVoxels();
    const size_t F = im.poses.size();
    const int lvl = data.rgbd_level;
    if (n == 0 || F == 0 || im.rgbd_pyr.size() != F || data.voxel_sh_coeffs.size() != n)
    {
        std::cerr << "Optimizer::optimize: inconsistent inputs (voxels " << n << ", poses " << F << ", pyramids " << im.rgbd_pyr.size() << ", sh "
                  << data.voxel_sh_coeffs.size() << ")" << std::endl;
        return false;
    }
    problem_info_.clear(); solver_info_.clear();

    // ---- flatten (iteration order == voxel_idx of optimizer.cpp:148-149)
    std::vector<int32_t> xyz(3 * n);
    std::vector<double> sdf0(n), sdf(n), alb(n), sh(9 * n, 0.0);
    std::vector<float> weight(n);
    std::vector<uint8_t> rgb(3 * n);
    size_t i = 0;
    for (auto it = grid->begin(); it != grid->end(); ++it, ++i)
    {
        const Vec3i& p = it->first; const VoxelSBR& v = it->second;
        xyz[3 * i] = p[0]; xyz[3 * i + 1] = p[1]; xyz[3 * i + 2] = p[2];
        sdf0[i] = v.sdf; sdf[i] = v.sdf_refined; alb[i] = v.albedo; weight[i] = v.weight;
        rgb[3 * i] = v.color[0]; rgb[3 * i + 1] = v.color[1]; rgb[3 * i + 2] = v.color[2];
        const VecXd& c = data.voxel_sh_coeffs[i];
        for (size_t k = 0; k < 9 && k < c.size(); ++k) sh[9 * i + k] = c[k];     // empty for out-of-shell voxels (never read)
    }
    const ImageF lum0 = im.rgbd_pyr[0].intensity(lvl);
    const int W = lum0.cols, H = lum0.rows;
    std::vector<float> lum(F * static_cast<size_t>(W) * H), depth(lum.size());
    for (size_t f = 0; f < F; ++f)
    {
        const ImageF l = im.rgbd_pyr[f].intensity(lvl), d = im.rgbd_pyr[f].depth(lvl);
        if (l.rows != H || l.cols != W || d.rows != H || d.cols != W) { std::cerr << "Optimizer::optimize: frame " << f << " has a different size" << std::endl; return false; }
        std::copy(l.data, l.data + static_cast<size_t>(W) * H, lum.begin() + f * static_cast<size_t>(W) * H);
        std::copy(d.data, d.data + static_cast<size_t>(W) * H, depth.begin() + f * static_cast<size_t>(W) * H);
    }
    std::vector<double> poses(6 * F);
    for (size_t f = 0; f < F; ++f) for (int k = 0; k < 6; ++k) poses[6 * f + k] = im.poses[f][k];

    // ---- engine
    I3DEngine* eng = nullptr;
    if (i3d_engine_create(device_, &eng) != 0) { std::cerr << "Optimizer::optimize: " << i3d_last_error(nullptr) << std::endl; return false; }
    auto fail = [&](const char* what) { std::cerr << "Optimizer::optimize: " << what << ": " << i3d_last_error(eng) << std::endl; i3d_engine_destroy(eng); return false; };
    if (i3d_upload_grid(eng, static_cast<int64_t>(n), xyz.data(), sdf0.data(), sdf.data(), alb.data(), weight.data(), rgb.data(), grid->voxelSize()) != 0) return fail("upload grid");
    if (i3d_upload_frames(eng, static_cast<int32_t>(F), W, H, lum.data(), depth.data(), pyramidLevelToScale(lvl)) != 0) return fail("upload frames");
    if (i3d_set_camera(eng, poses.data(), im.intrinsics.data(), im.distortion_coeffs.data()) != 0) return fail("set camera");
    if (i3d_set_sh(eng, sh.data()) != 0) return fail("set sh");

    bool ok = true;
    for (int itr = 0; itr < cfg_.iterations && ok; ++itr)
    {
        std::cout << "   iteration " << itr << " (grid level " << data.grid_level << ", pyramid level " << lvl << ")" << std::endl;
        colorization.reset(grid, im.intrinsics * pyramidLevelToScale(lvl), im.distortion_coeffs, W, H);
        // a fresh solver every outer iteration, like the reference (the trust-region radius restarts at the default, Q5)
        NLSSolver solver;
        solver.reset(4);
        if (std::getenv("I3D_HOST_DEBUG")) solver.setDebug(true);
        solver.setCostWeight(0, cfg_.lambda_g);
        solver.setCostWeight(1, computeVaryingLambda(itr, cfg_.iterations, cfg_.lambda_r0, cfg_.lambda_r1));
        solver.setCostWeight(2, computeVaryingLambda(itr, cfg_.iterations, cfg_.lambda_s0, cfg_.lambda_s1));
        solver.setCostWeight(3, cfg_.lambda_a);
        NLSSolver::Binding b;
        b.engine = eng; b.thres_shell = data.thres_shell;
        b.occlusion_distance = colorization.config().max_occlusion_distance;
        b.num_observations = static_cast<int>(colorization.config().max_num_observations);
        b.use_er = cfg_.lambda_r0 > 0.0 && cfg_.lambda_r1 > 0.0;
        b.use_es = cfg_.lambda_s0 > 0.0 && cfg_.lambda_s1 > 0.0;
        b.use_ea = cfg_.lambda_a > 0.0;
        b.fix_all_albedo = cfg_.lambda_a < 0.0;
        b.poses_begin = F ? im.poses[0].data() : nullptr; b.num_poses = F;
        b.intrinsics = im.intrinsics.data(); b.distortion = im.distortion_coeffs.data();
        solver.attach(b);
        if (!solver.buildProblem(true)) { ok = false; break; }
        if (cfg_.fix_poses) for (size_t f = 0; f < F; ++f) solver.fixParamBlock(im.poses[f].data());
        if (cfg_.fix_intrinsics) solver.fixParamBlock(im.intrinsics.data());
        if (cfg_.fix_distortion) solver.fixParamBlock(im.distortion_coeffs.data());
        if (!solver.solve(cfg_.lm_steps)) { ok = false; break; }       // no valid voxels => the engine returns without touching the state
        if (!solver.problemInfo().empty()) problem_info_.push_back(solver.problemInfo().back());
        if (!solver.solverInfo().empty()) solver_info_.push_back(solver.solverInfo().back());
    }

    // ---- write back in place
    if (ok)
    {
        double intr[4], dist[5];
        if (i3d_download_state(eng, sdf.data(), alb.data(), poses.data(), intr, dist) != 0) return fail("download");
        i = 0;
        for (auto it = grid->begin(); it != grid->end(); ++it, ++i) { it->second.sdf_refined = sdf[i]; it->second.albedo = alb[i]; }
        for (size_t f = 0; f < F; ++f) for (int k = 0; k < 6; ++k) im.poses[f][k] = poses[6 * f + k];
        for (int k = 0; k < 4; ++k) im.intrinsics[k] = intr[k];
        for (int k = 0; k < 5; ++k) im.distortion_coeffs[k] = dist[k];
    }
    else std::cerr << "Optimizer::optimize: engine error: " << i3d_last_error(eng) << std::endl;
    i3d_engine_destroy(eng);
    return ok;
}
} // namespace nv
