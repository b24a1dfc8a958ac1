/*
 * i3d_render.cu — the keyframe renderer (i3d_render.cuh) and the frame-to-model tracker (i3d_track.cuh), which marches the renderer's kernel
 * for its prediction: their kernels and the host code that sequences them (i3d_render.h, i3d_track.h).  Keeping them out of i3d_engine.cu
 * leaves the engine's device module as it is.
 */
#include <chrono>
#include <climits>
#include <cmath>
#include <cstring>
#include <optional>

#include "../../include/i3d_c_api.h"
#include "i3d_frames.h"
#include "i3d_render.cuh"
#include "i3d_track.cuh"

namespace i3d
{
namespace
{
// Bits of the renderer's brick bitmap above which the march visits every lattice sample instead (128 MiB)
constexpr int64_t kRenderBrickCap = 1ll << 30;

// Completes rg with the voxel box and (when it fits under kRenderBrickCap) the brick bitmap of its voxel set.  They are built, timed as
// "render_bricks", on the first call after the voxel set changed.
void add_voxel_box(RenderState& rs, Timing& tm, RenderGrid& rg, cudaStream_t st)
{
    if (!rs.box_ready)
    {
        Timer t(tm, st, "render_bricks");
        const int init[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
        rs.box_d.ensure(6);
        CK(cudaMemcpyAsync(rs.box_d.p, init, sizeof(init), cudaMemcpyHostToDevice, st));
        k_render_bounds<<<blocks_for(rg.g.n), kThreads, 0, st>>>(rg.g.n, rg.g.x, rg.g.y, rg.g.z, rs.box_d.p);
        CK(cudaMemcpyAsync(rs.box, rs.box_d.p, sizeof(rs.box), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        int64_t bits = 1;
        for (int d = 0; d < 3; ++d)
        {
            rs.blo[d] = rs.box[d];
            rs.bdim[d] = ((rs.box[3 + d] - rs.box[d]) >> 3) + 1;
            bits *= rs.bdim[d];
        }
        rs.have_bricks = bits <= kRenderBrickCap;
        if (rs.have_bricks)
        {
            const size_t words = static_cast<size_t>((bits + 31) >> 5);
            rs.bits.ensure(words);
            CK(cudaMemsetAsync(rs.bits.p, 0, words * sizeof(uint32_t), st));
            const BrickBox bb{{rs.blo[0], rs.blo[1], rs.blo[2]}, {rs.bdim[0], rs.bdim[1], rs.bdim[2]}};
            k_render_bricks<<<blocks_for(rg.g.n), kThreads, 0, st>>>(rg.g.n, rg.g.x, rg.g.y, rg.g.z, bb, rs.bits.p);
        }
        t.stop();
        rs.box_ready = true;
    }
    for (int d = 0; d < 3; ++d)
    {
        rg.lo[d] = static_cast<float>(rs.box[d]) * rg.g.voxel_size;
        rg.hi[d] = static_cast<float>(rs.box[3 + d]) * rg.g.voxel_size;
        rg.blo[d] = rs.blo[d]; rg.bdim[d] = rs.bdim[d];
    }
    rg.bricks = (rs.skip && rs.have_bricks) ? rs.bits.p : nullptr;
}

// The march of the installed grid; with mi also its model intensity plane from GridView::rgb
void march(const RenderGrid& rg, const RenderCam& cam, const RenderViews& rv, cudaStream_t st, float* mi = nullptr)
{
    const dim3 grid(rv.tiles_x, rv.tiles_y, rv.n), block(kRenderTile, kRenderTile);
    if (mi)
    {
        Colored<RenderGrid> cg{};
        static_cast<RenderGrid&>(cg) = rg;
        cg.rgb = rg.g.rgb; cg.out_mi = mi;
        k_render_march_color<<<grid, block, 0, st>>>(cg, cam, rv);
    }
    else k_render_march<<<grid, block, 0, st>>>(rg, cam, rv);
}

// out[n][V] = the fixed-order sums of the n views' partials [n][tiles][V]
template <int V>
void tile_sums(int n, int tiles, const double* partials, double* out, cudaStream_t st)
{
    k_tile_sums<V><<<blocks_for(static_cast<size_t>(n) * V), kThreads, 0, st>>>(n, tiles, partials, out);
}

// One view's kRenderStats sums
I3DRenderStats render_stats(const double* s)
{
    I3DRenderStats r;
    r.num_hit = static_cast<int64_t>(s[0]); r.num_observed = static_cast<int64_t>(s[1]);
    r.depth_count = static_cast<int64_t>(s[2]); r.photo_count = static_cast<int64_t>(s[3]);
    r.depth_abs = s[4]; r.depth_sq = s[5]; r.photo_abs = s[6]; r.photo_sq = s[7];
    return r;
}
} // namespace

void render::keyframes(RenderState& rs, Timing& tm, RenderGrid rg, const RenderCam& cam, const float* Rt, int n, const int32_t* ids, int W, int H,
                       const float* depth, const float* lum, int planes, bool photometric, I3DRenderStats* stats, cudaStream_t st)
{
    begin_timing(tm, {"render", "render_bricks", "render_samples"});
    rs.have_render = false;
    const size_t img = static_cast<size_t>(n) * W * H;
    if (planes & I3D_RENDER_DEPTH) rs.depth.ensure(img);
    if (planes & I3D_RENDER_NORMAL) rs.normal.ensure(3 * img);
    if (planes & I3D_RENDER_ALBEDO) rs.albedo.ensure(img);
    if (planes & I3D_RENDER_SHADING) rs.shading.ensure(img);
    if (planes & I3D_RENDER_INTENSITY) rs.intensity.ensure(img);
    const int tiles_x = (W + kRenderTile - 1) / kRenderTile, tiles_y = (H + kRenderTile - 1) / kRenderTile;
    rs.partials.ensure(static_cast<size_t>(n) * tiles_x * tiles_y * kRenderStats);
    rs.sums.ensure(static_cast<size_t>(n) * kRenderStats);
    rs.ids.ensure(n); rs.samples.ensure(1);
    CK(cudaMemcpyAsync(rs.ids.p, ids, n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(rs.samples.p, 0, sizeof(unsigned long long), st));
    {
        Timer t(tm, st, "render");
        add_voxel_box(rs, tm, rg, st);
        RenderViews rv;
        rv.n = n; rv.W = W; rv.H = H; rv.tiles_x = tiles_x; rv.tiles_y = tiles_y;
        rv.ids = rs.ids.p; rv.Rt = Rt; rv.depth = depth; rv.lum = lum;
        rv.out_depth = (planes & I3D_RENDER_DEPTH) ? rs.depth.p : nullptr;
        rv.out_normal = (planes & I3D_RENDER_NORMAL) ? rs.normal.p : nullptr;
        rv.out_albedo = (planes & I3D_RENDER_ALBEDO) ? rs.albedo.p : nullptr;
        rv.out_shading = (planes & I3D_RENDER_SHADING) ? rs.shading.p : nullptr;
        rv.out_intensity = (planes & I3D_RENDER_INTENSITY) ? rs.intensity.p : nullptr;
        rv.partials = rs.partials.p; rv.samples = rs.samples.p; rv.photometric = photometric ? 1 : 0;
        march(rg, cam, rv, st);
        tile_sums<kRenderStats>(n, tiles_x * tiles_y, rs.partials.p, rs.sums.p, st);
    }
    std::vector<double> sums(static_cast<size_t>(n) * kRenderStats);
    unsigned long long samples = 0;
    CK(cudaMemcpyAsync(sums.data(), rs.sums.p, sums.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&samples, rs.samples.p, sizeof(samples), cudaMemcpyDeviceToHost, st));
    collect_kernel_times(tm, st);
    CK(cudaGetLastError());
    tm.phases["render_samples"].count = static_cast<int64_t>(samples);
    if (stats)
        for (int i = 0; i < n; ++i) stats[i] = render_stats(sums.data() + static_cast<size_t>(i) * kRenderStats);
    rs.have_render = true; rs.n = n; rs.planes = planes;
}

namespace
{
// The phase names of one tracking pass (whole: nullptr = not timed as a whole)
struct TrackPhases
{
    const char* whole; const char* predict; const char* pyramid; const char* icp; const char* correspondences;
    const char* color; const char* photo_correspondences; const char* reference;
};
constexpr TrackPhases kTrackPhases{"track", "track_predict", "track_pyramid", "track_icp", "track_correspondences", "track_color",
                                   "track_photo_correspondences", "track_reference"};
constexpr TrackPhases kOdometryPhases{nullptr, "odometry_predict", "odometry_icp", "odometry_icp", "odometry_correspondences", "odometry_icp",
                                      "odometry_photo_correspondences", "odometry_icp"};

// The tracker's passes over ids[0..n), shared by the grid and the fusion volume: prepare() (false: stop, nothing tracked) runs once
// after the uploads, predict(cam, rv, mi) marches a chunk's prediction into rv, and with mi != nullptr the model intensity plane into mi.
// pose_cw_out [n][12] (may be nullptr): the tracked camera -> world poses.  col: the photometric term (nullptr: depth only); with its
// reference the plain march, then per pass the references' pyramids and k_track_ref_model per level, timed as ph.reference; with its
// norm_radius > 0 also both intensity pyramids through k_track_local_norm (DESIGN.md §6r).  Returns false when prepare() stopped the call.
template <class Prepare, class Predict>
bool track_passes(TrackScratch& ts, Timing& tm, const TrackPhases& ph, Prepare&& prepare, Predict&& predict, const I3DFusionCamera& dc,
                  const float* store_depth, int store_F, int n, const int32_t* ids, const double* pose_in, const I3DTrackParams& P, const int* Wl,
                  const int* Hl, double* pose_out, double* pose_cw_out, I3DTrackInfo* info, cudaStream_t st, const TrackColor* col)
{
    const int L = P.num_levels, W = dc.width, H = dc.height, C = std::min<int>(n, I3D_TRACK_CHUNK);
    const size_t img = static_cast<size_t>(W) * H;
    const bool ref = col && col->ref_ids;
    const int norm_r = ref ? col->P->norm_radius : 0;       // DESIGN.md §6r: > 0 normalises both intensity pyramids
    const int tiles_x = (W + kRenderTile - 1) / kRenderTile, tiles_y = (H + kRenderTile - 1) / kRenderTile;
    static_assert(kRenderTile == kTrackTile, "the prediction and the rows share the level-0 tile grid");
    ts.n = 0;
    ts.ids.ensure(n); ts.pose_in.ensure(12 * static_cast<size_t>(n)); ts.state.ensure(n);
    ts.sys.ensure(static_cast<size_t>(n) * kTrackVals); ts.rd_sums.ensure(static_cast<size_t>(n) * kRenderStats);
    ts.rt.ensure(12 * static_cast<size_t>(store_F)); ts.counters.ensure(3);
    ts.rd_partials.ensure(static_cast<size_t>(C) * tiles_x * tiles_y * kRenderStats);
    ts.partials.ensure(static_cast<size_t>(C) * tiles_x * tiles_y * kTrackVals); ts.sums.ensure(static_cast<size_t>(C) * kTrackVals);
    ts.pdepth.ensure(C * img); ts.pnrm.ensure(3 * C * img); ts.mask.ensure(C * img);
    for (int l = 0; l < L; ++l)
    {
        const size_t c = static_cast<size_t>(C) * Wl[l] * Hl[l];
        ts.depth[l].ensure(c); ts.nrm[l].ensure(3 * c);
        if (col) { ts.inten[l].ensure(c); ts.gx[l].ensure(c); ts.gy[l].ensure(c); }
        if (ref) { ts.ref_inten[l].ensure(c); ts.ref_depth[l].ensure(c); }
        if (norm_r > 0) { ts.raw_inten[l].ensure(c); ts.raw_ref_inten[l].ensure(c); }
        if (ref && l > 0) ts.ref_model[l].ensure(C * img);
    }
    std::vector<float> hr(ref ? 12 * static_cast<size_t>(n) : 0);      // the reference poses in float, by call order
    if (ref)
    {
        for (size_t i = 0; i < hr.size(); ++i) hr[i] = static_cast<float>(col->ref_pose[i]);
        ts.ref_ids.ensure(n); ts.ref_rt.ensure(hr.size());
        CK(cudaMemcpyAsync(ts.ref_ids.p, col->ref_ids, n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(ts.ref_rt.p, hr.data(), hr.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    if (col)
    {
        ts.pint.ensure(C * img); ts.iota.ensure(C);
        ts.partials_c.ensure(static_cast<size_t>(C) * tiles_x * tiles_y * kTrackVals);
        ts.sums_c.ensure(static_cast<size_t>(C) * kTrackVals); ts.sums_comb.ensure(static_cast<size_t>(C) * kTrackVals);
        ts.sys_c.ensure(static_cast<size_t>(n) * kTrackVals); ts.cstate.ensure(n);
        std::vector<int32_t> iota(C);
        for (int k = 0; k < C; ++k) iota[k] = k;
        CK(cudaMemcpyAsync(ts.iota.p, iota.data(), C * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(ts.cstate.p, 0, n * sizeof(TrackColorState), st));
    }
    // the input poses in float, scattered by sensor id: the march reads Rt + 12 * id
    std::vector<float> hrt(12 * static_cast<size_t>(store_F), 0.0f);
    for (int k = 0; k < n; ++k)
        for (int i = 0; i < 12; ++i) hrt[12 * static_cast<size_t>(ids[k]) + i] = static_cast<float>(pose_in[12 * static_cast<size_t>(k) + i]);
    CK(cudaMemcpyAsync(ts.ids.p, ids, n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ts.pose_in.p, pose_in, 12 * static_cast<size_t>(n) * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ts.rt.p, hrt.data(), hrt.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(ts.counters.p, 0, 3 * sizeof(unsigned long long), st));
    int total_iters = 0;
    for (int l = 0; l < L; ++l) total_iters += P.iterations[l];
    TrackCam cam[kTrackMaxLevels];
    for (int l = 0; l < L; ++l)
    {
        const double s = std::ldexp(1.0, -l);       // the pyramid scale, as select_cam applies pyr_scale
        cam[l] = TrackCam{Wl[l], Hl[l], static_cast<float>(dc.fx * s), static_cast<float>(dc.fy * s), static_cast<float>(dc.cx * s),
                          static_cast<float>(dc.cy * s)};
    }
    std::optional<Timer> whole;
    if (ph.whole) whole.emplace(tm, st, ph.whole);
    if (!prepare()) return false;
    RenderCam rcam{};
    rcam.fx = dc.fx; rcam.fy = dc.fy; rcam.cx = dc.cx; rcam.cy = dc.cy; rcam.dist_zero = 1;
    k_track_init<<<blocks_for(n, 64), 64, 0, st>>>(n, ts.pose_in.p, ts.state.p);
    const float max_dist_sq = P.max_distance * P.max_distance;
    int m = 0;
    // a chunk's pyramid lv: the stored depth of device ids then frames::depthdown, or frames::sensor_intensity of host ids then pyrdown
    auto depth_pyramid = [&](const int32_t* ids_dev, Dev<float>* lv) {
        k_track_gather<<<dim3(blocks_for(img), m), kThreads, 0, st>>>(m, W, H, ids_dev, store_depth, lv[0].p);
        for (int l = 1; l < L; ++l) frames::depthdown(m, Wl[l - 1], Hl[l - 1], lv[l - 1].p, lv[l].p, st);
    };
    // with norm_r > 0 the raw pyramid goes to raw (each level the pyrdown of the raw level above) and k_track_local_norm writes lv
    auto intensity_pyramid = [&](const int32_t* ids_host, Dev<float>* lv, Dev<float>* raw) {
        Dev<float>* py = norm_r > 0 ? raw : lv;
        frames::sensor_intensity(*col->ss, m, ids_host, ts.iota.p, ts.lum_c, py[0].p, st);
        for (int l = 1; l < L; ++l) frames::pyrdown(m, Wl[l - 1], Hl[l - 1], py[l - 1].p, py[l].p, st);
        for (int l = 0; l < L && norm_r > 0; ++l)
        {
            const int blocks = ((Wl[l] + kTrackLniTileW - 1) / kTrackLniTileW) * ((Hl[l] + kTrackLniTileH - 1) / kTrackLniTileH);
            Timer tk(tm, st, "track_local_norm", 1);
            k_track_local_norm<<<dim3(blocks, m), dim3(kTrackLniTileW, kTrackLniTileH), 0, st>>>(Wl[l], Hl[l], norm_r, col->P->norm_eps, raw[l].p,
                                                                                                 lv[l].p);
        }
    };
    for (int c0 = 0; c0 < n; c0 += C)
    {
        m = std::min(C, n - c0);
        const int32_t* ids_d = ts.ids.p + c0;
        {
            Timer t(tm, st, ph.predict);
            RenderViews rv{};
            rv.n = m; rv.W = W; rv.H = H; rv.tiles_x = tiles_x; rv.tiles_y = tiles_y;
            rv.ids = ids_d; rv.Rt = ts.rt.p; rv.depth = store_depth; rv.lum = nullptr;
            rv.out_depth = ts.pdepth.p; rv.out_normal = ts.pnrm.p;
            rv.partials = ts.rd_partials.p; rv.samples = ts.counters.p + 1; rv.photometric = 0;
            predict(rcam, rv, col && !ref ? ts.pint.p : nullptr);
            tile_sums<kRenderStats>(m, tiles_x * tiles_y, ts.rd_partials.p, ts.rd_sums.p + static_cast<size_t>(c0) * kRenderStats, st);
        }
        {
            Timer t(tm, st, ph.pyramid);
            depth_pyramid(ids_d, ts.depth);
            for (int l = 0; l < L; ++l)
                k_track_normals<<<dim3(blocks_for(static_cast<size_t>(Wl[l]) * Hl[l]), m), kThreads, 0, st>>>(cam[l], ts.depth[l].p, ts.nrm[l].p);
        }
        if (col)
        {
            // the frame intensity pyramid in the depth camera and its gradients
            Timer t(tm, st, ph.color);
            intensity_pyramid(ids + c0, ts.inten, ts.raw_inten);
            for (int l = 0; l < L; ++l)
                k_track_grad<<<dim3(blocks_for(static_cast<size_t>(Wl[l]) * Hl[l]), m), kThreads, 0, st>>>(cam[l], ts.inten[l].p, ts.gx[l].p, ts.gy[l].p);
        }
        if (ref)
        {
            // the references' intensity and depth pyramids by the frame's own rules, then each level's model plane
            Timer t(tm, st, ph.reference);
            intensity_pyramid(col->ref_ids + c0, ts.ref_inten, ts.raw_ref_inten);
            depth_pyramid(ts.ref_ids.p + c0, ts.ref_depth);
            TrackRef tf{};
            tf.pcam = cam[0]; tf.pdepth = ts.pdepth.p; tf.ids = ids_d; tf.rt_in = ts.rt.p; tf.ref_rt = ts.ref_rt.p + 12 * static_cast<size_t>(c0);
            tf.max_distance = P.max_distance;
            for (int l = 0; l < L; ++l)
            {
                tf.cam = cam[l]; tf.step = 1 << l; tf.inten = ts.ref_inten[l].p; tf.depth = ts.ref_depth[l].p;
                tf.model = l == 0 ? ts.pint.p : ts.ref_model[l].p;
                Timer tk(tm, st, "track_ref_model", 1);
                k_track_ref_model<<<dim3(blocks_for(static_cast<size_t>(Wl[l]) * Hl[l]), m), kThreads, 0, st>>>(tf);
            }
        }
        {
            Timer t(tm, st, ph.icp);
            CK(cudaMemsetAsync(ts.mask.p, 0, m * img, st));
            TrackRows tr{};
            tr.pcam = cam[0]; tr.pdepth = ts.pdepth.p; tr.pnrm = ts.pnrm.p; tr.ids = ids_d; tr.rt_in = ts.rt.p;
            tr.state = ts.state.p + c0; tr.max_dist_sq = max_dist_sq; tr.min_cos = P.min_normal_cos;
            tr.use_cos = P.min_normal_cos > -1.0f ? 1 : 0; tr.partials = ts.partials.p;
            TrackPhoto tp{};
            if (col)
            {
                tp.pcam = cam[0]; tp.pdepth = ts.pdepth.p; tp.pint = ts.pint.p; tp.ids = ids_d; tp.rt_in = ts.rt.p; tp.state = ts.state.p + c0;
                tp.max_distance = P.max_distance; tp.max_diff = col->P->max_color_diff;
                tp.min_grad_sq = col->P->min_color_gradient * col->P->min_color_gradient; tp.partials = ts.partials_c.p;
            }
            auto system = [&](int l, int solve) {
                tr.cam = cam[l]; tr.depth = ts.depth[l].p; tr.nrm = ts.nrm[l].p; tr.mask = l == 0 ? ts.mask.p : nullptr;
                tr.tiles_x = (Wl[l] + kTrackTile - 1) / kTrackTile; tr.tiles_y = (Hl[l] + kTrackTile - 1) / kTrackTile;
                {
                    Timer tk(tm, st, "k_track_rows", 1);
                    k_track_rows<<<dim3(tr.tiles_x, tr.tiles_y, m), dim3(kTrackTile, kTrackTile), 0, st>>>(tr);
                }
                tile_sums<kTrackVals>(m, tr.tiles_x * tr.tiles_y, ts.partials.p, ts.sums.p, st);
                const double* S = ts.sums.p;
                if (col)
                {
                    tp.cam = cam[l]; tp.step = 1 << l; tp.inten = ts.inten[l].p; tp.gx = ts.gx[l].p; tp.gy = ts.gy[l].p; tp.depth = ts.depth[l].p;
                    if (ref) tp.pint = l == 0 ? ts.pint.p : ts.ref_model[l].p;
                    tp.tiles_x = tr.tiles_x; tp.tiles_y = tr.tiles_y;
                    {
                        Timer tk(tm, st, "track_photo_rows", 1);
                        k_track_photo_rows<<<dim3(tp.tiles_x, tp.tiles_y, m), dim3(kTrackTile, kTrackTile), 0, st>>>(tp);
                    }
                    tile_sums<kTrackVals>(m, tp.tiles_x * tp.tiles_y, ts.partials_c.p, ts.sums_c.p, st);
                    const double w = static_cast<double>(col->P->weight[l]);
                    k_track_combine<<<blocks_for(m, 64), 64, 0, st>>>(m, w * w, ts.sums.p, ts.sums_c.p, ts.state.p + c0, ts.cstate.p + c0, ts.sums_comb.p,
                                                                      ts.sys_c.p + static_cast<size_t>(c0) * kTrackVals, ts.counters.p + 2);
                    S = ts.sums_comb.p;
                }
                k_track_solve<<<blocks_for(m, 64), 64, 0, st>>>(m, S, ts.state.p + c0, ts.sys.p + static_cast<size_t>(c0) * kTrackVals,
                                                                P.min_correspondences, solve, ts.counters.p);
            };
            for (int l = L - 1; l >= 0; --l)
                for (int it = 0; it < P.iterations[l]; ++it) system(l, 1);
            if (total_iters == 0) system(0, 0);        // no update: the level-0 system at the input pose
        }
    }
    std::vector<TrackState> hs(n);
    std::vector<double> rs_sums(static_cast<size_t>(n) * kRenderStats);
    std::vector<TrackColorState> hc(col ? n : 0);
    unsigned long long counters[3] = {0, 0, 0};
    CK(cudaMemcpyAsync(hs.data(), ts.state.p, n * sizeof(TrackState), cudaMemcpyDeviceToHost, st));
    if (col) CK(cudaMemcpyAsync(hc.data(), ts.cstate.p, n * sizeof(TrackColorState), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(rs_sums.data(), ts.rd_sums.p, rs_sums.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(counters, ts.counters.p, sizeof(counters), cudaMemcpyDeviceToHost, st));
    if (whole) whole->stop();
    collect_kernel_times(tm, st);
    CK(cudaGetLastError());
    tm.phases[ph.correspondences].count += static_cast<int64_t>(counters[0]);
    if (col) tm.phases[ph.photo_correspondences].count += static_cast<int64_t>(counters[2]);
    for (int k = 0; k < n; ++k)
    {
        std::memcpy(pose_out + 12 * static_cast<size_t>(k), hs[k].w2c, 12 * sizeof(double));
        if (pose_cw_out) std::memcpy(pose_cw_out + 12 * static_cast<size_t>(k), hs[k].T, 12 * sizeof(double));
        if (col && col->info) col->info[k] = I3DTrackColorInfo{hc[k].first_rows, hc[k].first_sq, hc[k].last_rows, hc[k].last_sq};
        if (!info) continue;
        I3DTrackInfo r{};
        r.status = hs[k].status; r.iterations = hs[k].iterations; r.correspondences = hs[k].correspondences;
        r.residual_sq = hs[k].residual_sq; r.update_norm = hs[k].update_norm;
        r.initial = render_stats(rs_sums.data() + static_cast<size_t>(k) * kRenderStats);
        info[k] = r;
    }
    ts.n = n; ts.levels = L; ts.last_m = m; ts.color = col != nullptr; ts.reference = ref;
    for (int l = 0; l < L; ++l) { ts.W[l] = Wl[l]; ts.H[l] = Hl[l]; }
    return true;
}


// Completes lg from the fusion volume fv: the box of its voxels with weight > 0 and, when skip and it fits under kRenderBrickCap, their
// brick bitmap; timed as `phase`.  The box read synchronises.  Returns false when no voxel has weight > 0.
bool live_box(TrackScratch& ts, Timing& tm, const char* phase, const FuseView& fv, float voxel_size, bool skip, LiveGrid& lg, cudaStream_t st)
{
    Timer t(tm, st, phase);
    int box[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
    ts.live_box.ensure(6);
    CK(cudaMemcpyAsync(ts.live_box.p, box, sizeof(box), cudaMemcpyHostToDevice, st));
    if (fv.n > 0) k_live_bounds<<<blocks_for(fv.n), kThreads, 0, st>>>(fv.n, fv.x, fv.y, fv.z, fv.weight, ts.live_box.p);
    CK(cudaMemcpyAsync(box, ts.live_box.p, sizeof(box), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (box[0] > box[3]) return false;
    lg.v = fv; lg.voxel_size = voxel_size; lg.bricks = nullptr;
    int64_t bits = 1;
    for (int d = 0; d < 3; ++d)
    {
        lg.lo[d] = static_cast<float>(box[d]) * voxel_size;
        lg.hi[d] = static_cast<float>(box[3 + d]) * voxel_size;
        lg.blo[d] = box[d];
        lg.bdim[d] = ((box[3 + d] - box[d]) >> 3) + 1;
        bits *= lg.bdim[d];
    }
    if (skip && bits <= kRenderBrickCap)
    {
        const size_t words = static_cast<size_t>((bits + 31) >> 5);
        ts.live_bits.ensure(words);
        CK(cudaMemsetAsync(ts.live_bits.p, 0, words * sizeof(uint32_t), st));
        const BrickBox bb{{lg.blo[0], lg.blo[1], lg.blo[2]}, {lg.bdim[0], lg.bdim[1], lg.bdim[2]}};
        k_live_bricks<<<blocks_for(fv.n), kThreads, 0, st>>>(fv.n, fv.x, fv.y, fv.z, fv.weight, bb, ts.live_bits.p);
        lg.bricks = ts.live_bits.p;
    }
    return true;
}

// The march of the volume in progress; with mi also its model intensity plane from the voxel colours rgb
void march_live(const LiveGrid& lg, const RenderCam& cam, const RenderViews& rv, const uchar4* rgb, float* mi, cudaStream_t st)
{
    const dim3 grid(rv.tiles_x, rv.tiles_y, rv.n), block(kRenderTile, kRenderTile);
    if (mi)
    {
        Colored<LiveGrid> cg{};
        static_cast<LiveGrid&>(cg) = lg;
        cg.rgb = rgb; cg.out_mi = mi;
        k_render_march_live_color<<<grid, block, 0, st>>>(cg, cam, rv);
    }
    else k_render_march_live<<<grid, block, 0, st>>>(lg, cam, rv);
}

// Poses R row-major | t in double, every sum left to right as tests/test_odometry.py restates them.  The inverse is tr_inverse's.
void pose_inverse(const double* T, double* out)
{
    for (int i = 0; i < 3; ++i)
    {
        for (int j = 0; j < 3; ++j) out[3 * i + j] = T[3 * j + i];
        out[9 + i] = -((T[i] * T[9] + T[3 + i] * T[10]) + T[6 + i] * T[11]);
    }
}

// A . B = [R_A R_B | R_A t_B + t_A]
void pose_compose(const double* A, const double* B, double* out)
{
    for (int a = 0; a < 3; ++a)
    {
        for (int c = 0; c < 3; ++c) out[3 * a + c] = (A[3 * a] * B[c] + A[3 * a + 1] * B[3 + c]) + A[3 * a + 2] * B[6 + c];
        out[9 + a] = ((A[3 * a] * B[9] + A[3 * a + 1] * B[10]) + A[3 * a + 2] * B[11]) + A[9 + a];
    }
}
} // namespace

void track::sensor_frames(TrackScratch& ts, RenderState& rs, Timing& tm, RenderGrid rg, const I3DFusionCamera& dc, const float* store_depth,
                          int store_F, int n, const int32_t* ids, const double* pose_in, const I3DTrackParams& P, const int* Wl, const int* Hl,
                          double* pose_out, I3DTrackInfo* info, cudaStream_t st, const TrackColor* col)
{
    begin_timing(tm, {"track", "track_predict", "track_pyramid", "track_icp", "track_correspondences", "track_color", "track_photo_rows",
                      "track_photo_correspondences", "track_reference", "track_ref_model", "track_local_norm"});
    track_passes(
        ts, tm, kTrackPhases, [&]() { add_voxel_box(rs, tm, rg, st); return true; },
        [&](const RenderCam& cam, const RenderViews& rv, float* mi) { march(rg, cam, rv, st, mi); }, dc, store_depth, store_F, n, ids, pose_in, P,
        Wl, Hl, pose_out, nullptr, info, st, col);
}

int track::fusion_frames(TrackScratch& ts, const FusionState& fs, bool skip, Timing& tm, const SensorStore& ss, int n, const int32_t* ids,
                         const double* pose_in, const I3DTrackParams& P, const int* Wl, const int* Hl, double* pose_out, I3DTrackInfo* info, cudaStream_t st,
                         const TrackColor* col)
{
    begin_timing(tm, {"track", "track_predict", "track_pyramid", "track_icp", "track_correspondences", "track_bricks", "track_color",
                      "track_photo_rows", "track_photo_correspondences", "track_reference", "track_ref_model", "track_local_norm"});
    LiveGrid lg{};
    const bool ok = track_passes(
        ts, tm, kTrackPhases, [&]() { return live_box(ts, tm, "track_bricks", fusion::view(fs), fs.p.voxel_size, skip, lg, st); },
        [&](const RenderCam& cam, const RenderViews& rv, float* mi) { march_live(lg, cam, rv, fs.rgb.p, mi, st); }, ss.dcam, ss.depth.p, ss.F, n,
        ids, pose_in, P, Wl, Hl, pose_out, nullptr, info, st, col);
    if (!ok) collect_kernel_times(tm, st);
    return ok ? 0 : 1;
}

int track::odometry(TrackScratch& ts, FusionState& fs, bool skip, Timing& tm, const SensorStore& ss, int n, const int32_t* ids, const double* pose_first,
                    const I3DTrackParams& P, const int* Wl, const int* Hl, double* pose_out, I3DTrackInfo* info, std::string& error, cudaStream_t st,
                    const TrackColor* col, bool reference)
{
    const auto t0 = std::chrono::steady_clock::now();
    for (const char* nm : {"odometry", "odometry_predict", "odometry_icp", "odometry_correspondences", "odometry_photo_correspondences", "track_photo_rows",
                           "track_ref_model", "track_local_norm"})
        tm.phases.erase(nm);
    // the motion state and the reference, kept here while fusion::integrate (which clears fs's) runs
    int motion = pose_first ? 0 : fs.motion;
    double prev[12], last[12];
    std::memcpy(prev, fs.motion_T[0], sizeof(prev)); std::memcpy(last, fs.motion_T[1], sizeof(last));
    int32_t ref_id = pose_first ? -1 : fs.ref_id;
    double ref_T[12];
    std::memcpy(ref_T, fs.ref_T, sizeof(ref_T));
    for (int k = 0; k < n; ++k)
    {
        // the guess: T_cw(k) = T_cw(k-1) . (T_cw(k-2)^-1 . T_cw(k-1)), or T_cw(k-1) with one previous pose
        double T[12], W[12];
        if (k == 0 && pose_first)
        {
            std::memcpy(W, pose_first, sizeof(W));
            pose_inverse(W, T);
        }
        else
        {
            if (motion == 1) std::memcpy(T, last, sizeof(T));
            else
            {
                double ip[12], d[12];
                pose_inverse(prev, ip);
                pose_compose(ip, last, d);
                pose_compose(last, d, T);
            }
            pose_inverse(T, W);
        }
        begin_timing(tm, {});
        I3DTrackInfo r{};
        I3DTrackColorInfo rc{};
        double Tt[12], Wt[12];
        const double* Ti = nullptr;
        const double* Wi = nullptr;
        LiveGrid lg{};
        if (!live_box(ts, tm, "odometry_predict", fusion::view(fs), fs.p.voxel_size, skip, lg, st))
        {
            collect_kernel_times(tm, st);
            r.status = I3D_TRACK_ANCHORED;
            Ti = T; Wi = W;
        }
        else
        {
            TrackColor c1{};
            double ref_W[12];
            if (col) c1 = TrackColor{col->P, col->ss, &rc};
            if (reference && ref_id >= 0)
            {
                pose_inverse(ref_T, ref_W);
                c1.ref_ids = &ref_id; c1.ref_pose = ref_W;
            }
            const bool with_color = col && (!reference || ref_id >= 0);          // no reference yet: depth alone
            track_passes(
                ts, tm, kOdometryPhases, []() { return true; },
                [&](const RenderCam& cam, const RenderViews& rv, float* mi) { march_live(lg, cam, rv, fs.rgb.p, mi, st); }, ss.dcam, ss.depth.p, ss.F,
                1, ids + k, W, P, Wl, Hl, Wt, Tt, &r, st, with_color ? &c1 : nullptr);
            if (r.status == I3D_TRACK_OK) { Ti = Tt; Wi = Wt; }
        }
        if (Ti)
        {
            float c2w[12], w2c[12];
            for (int i = 0; i < 12; ++i) { c2w[i] = static_cast<float>(Ti[i]); w2c[i] = static_cast<float>(Wi[i]); }
            if (fusion::integrate(fs, tm, 1, ss.dcam, ss.depth.p, ss.ccam, ss.bgr.p, ids + k, c2w, w2c, error, st)) return 1;
            std::memcpy(prev, last, sizeof(prev)); std::memcpy(last, Ti, sizeof(last));
            motion = std::min(motion + 1, 2);
            ref_id = ids[k];
            std::memcpy(ref_T, Ti, sizeof(ref_T));
        }
        else
        {
            // not integrated: the velocity is zero from the last integrated pose (the guess when this state has none)
            if (motion == 0) std::memcpy(last, T, sizeof(last));
            motion = 1;
        }
        fs.motion = motion;
        std::memcpy(fs.motion_T[0], prev, sizeof(prev)); std::memcpy(fs.motion_T[1], last, sizeof(last));
        fs.ref_id = ref_id;
        std::memcpy(fs.ref_T, ref_T, sizeof(ref_T));
        std::memcpy(pose_out + 12 * static_cast<size_t>(k), Wi ? Wi : W, 12 * sizeof(double));
        if (info) info[k] = r;
        if (col && col->info) col->info[k] = rc;
    }
    tm.phases["odometry"].ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    tm.phases["odometry"].count += 1;
    return 0;
}

} // namespace i3d
