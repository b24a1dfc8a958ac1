/*
 * i3d_distance.cu — the distance between the resident mesh and a reference mesh, and the registration of the reference to the resident
 * mesh: their kernels (i3d_distance.cuh, i3d_register.cuh) and the host code that sizes the search grids and launches them
 * (i3d_distance.h).  The registration's solve and pose update are the tracker's kernels, launched through track::pose_init / pose_step
 * (i3d_render.cu).  Keeping them out of i3d_engine.cu leaves the engine's device module as it is.
 */
#include <climits>
#include <cstdarg>
#include <cmath>
#include <cstdio>
#include <cstring>

#include "i3d_distance.cuh"
#include "i3d_register.cuh"

#include <cub/device/device_scan.cuh>

namespace i3d
{
namespace distance
{
namespace
{
struct AddI64 { __device__ __forceinline__ int64_t operator()(int64_t a, int64_t b) const { return a + b; } };

std::string format(const char* fmt, ...)
{
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    return buf;
}

void side_info(const double* s, const DistGrid& g, int64_t samples, int64_t entries, int nt, I3DDistanceSide& o)
{
    o.num_samples = samples;
    o.num_matched = static_cast<int64_t>(s[1]);
    o.area = s[2]; o.unmatched_area = s[3];
    o.mean = s[0] > 0.0 ? s[4] / s[0] : 0.0;
    o.rms = s[0] > 0.0 ? std::sqrt(s[5] / s[0]) : 0.0;
    o.max = s[6];
    for (int k = 0; k < nt; ++k) o.fraction[k] = s[2] > 0.0 ? s[8 + k] / s[2] : 0.0;
    o.point_triangle_tests = static_cast<int64_t>(s[7]);
    o.cell_size = g.h;
    for (int k = 0; k < 3; ++k) o.grid[k] = g.n[k];
    o.num_cells = static_cast<int64_t>(g.n[0]) * g.n[1] * g.n[2];
    o.num_cell_entries = entries;
}
} // namespace

bool plan(DistGridScratch& ds, const DistMesh& t, float cell_size, float max_distance, DistGrid& g, int64_t& entries, double* bounds, std::string& error,
          cudaStream_t st)
{
    const unsigned nb = blocks_for(static_cast<size_t>(t.F));
    ds.partials.ensure(static_cast<size_t>(nb) * kDistBounds);
    k_dist_bounds<<<nb, kThreads, 0, st>>>(t, ds.partials.p);
    std::vector<double> h(static_cast<size_t>(nb) * kDistBounds);
    CK(cudaMemcpyAsync(h.data(), ds.partials.p, h.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    double b[kDistBounds];
    for (int j = 0; j < kDistBounds; ++j) b[j] = h[j];
    for (unsigned i = 1; i < nb; ++i)
        for (int j = 0; j < kDistBounds; ++j) b[j] = j < 6 ? std::max(b[j], h[i * kDistBounds + j]) : b[j] + h[i * kDistBounds + j];
    if (bounds)
        for (int k = 0; k < 3; ++k) { bounds[k] = -b[k]; bounds[3 + k] = b[3 + k]; }
    const double mean_edge = b[6] / (3.0 * static_cast<double>(t.F));
    float cell = cell_size > 0.0f ? cell_size : static_cast<float>(2.0 * mean_edge);
    if (!(cell > 0.0f)) cell = max_distance;          // every face of the target is a point
    std::memset(&g, 0, sizeof(g));
    g.h = cell;
    double extent = 0.0, mag = 0.0, cells = 1.0;
    for (int k = 0; k < 3; ++k)
    {
        const float lo = static_cast<float>(-b[k]) - max_distance, hi = static_cast<float>(b[3 + k]) + max_distance;
        const double n = std::floor((static_cast<double>(hi) - lo) / cell) + 1.0;
        cells *= n;
        g.lo[k] = lo;
        g.n[k] = n < static_cast<double>(I3D_DISTANCE_MAX_CELLS) ? static_cast<int>(n) : static_cast<int>(I3D_DISTANCE_MAX_CELLS);
        extent = std::max(extent, static_cast<double>(hi) - lo);
        mag = std::max(mag, std::max(std::fabs(static_cast<double>(lo)), std::fabs(static_cast<double>(hi))));
    }
    if (cells > static_cast<double>(I3D_DISTANCE_MAX_CELLS))
    {
        error = format("a search grid of %.0f cells at cell_size %g m exceeds I3D_DISTANCE_MAX_CELLS (%lld); use a larger cell_size", cells,
                       static_cast<double>(cell), static_cast<long long>(I3D_DISTANCE_MAX_CELLS));
        return false;
    }
    g.margin = std::ldexp(mag + extent + cell, -16);
    ds.counter.ensure(1);
    CK(cudaMemsetAsync(ds.counter.p, 0, sizeof(unsigned long long), st));
    k_dist_entries<<<nb, kThreads, 0, st>>>(t, g, ds.counter.p);
    unsigned long long e = 0;
    CK(cudaMemcpyAsync(&e, ds.counter.p, sizeof(e), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    entries = static_cast<int64_t>(e);
    if (entries > I3D_DISTANCE_MAX_CELL_ENTRIES)
    {
        error = format("a search grid of %lld (face, cell) entries at cell_size %g m exceeds I3D_DISTANCE_MAX_CELL_ENTRIES (%lld); use a larger cell_size",
                       static_cast<long long>(entries), static_cast<double>(cell), static_cast<long long>(I3D_DISTANCE_MAX_CELL_ENTRIES));
        return false;
    }
    return true;
}

// cell_count ends as the per-cell counts again
void build(DistGridScratch& ds, const DistMesh& t, DistGrid& g, int64_t entries, cudaStream_t st)
{
    const size_t cells = static_cast<size_t>(g.n[0]) * g.n[1] * g.n[2];
    ds.cell_count.ensure(cells); ds.cell_off.ensure(cells); ds.cell_faces.ensure(static_cast<size_t>(entries));
    const unsigned nb = blocks_for(static_cast<size_t>(t.F));
    CK(cudaMemsetAsync(ds.cell_count.p, 0, cells * sizeof(int32_t), st));
    k_dist_insert<<<nb, kThreads, 0, st>>>(t, g, nullptr, ds.cell_count.p, nullptr);
    size_t bytes = 0;
    CK(cub::DeviceScan::ExclusiveScan(nullptr, bytes, static_cast<const int32_t*>(ds.cell_count.p), ds.cell_off.p, AddI64(), static_cast<int64_t>(0),
                                      static_cast<int64_t>(cells), st));
    ds.cub.ensure(bytes);
    CK(cub::DeviceScan::ExclusiveScan(static_cast<void*>(ds.cub.p), bytes, static_cast<const int32_t*>(ds.cell_count.p), ds.cell_off.p, AddI64(),
                                      static_cast<int64_t>(0), static_cast<int64_t>(cells), st));
    CK(cudaMemsetAsync(ds.cell_count.p, 0, cells * sizeof(int32_t), st));
    k_dist_insert<<<nb, kThreads, 0, st>>>(t, g, ds.cell_off.p, ds.cell_count.p, ds.cell_faces.p);
    g.off = ds.cell_off.p; g.cnt = ds.cell_count.p; g.faces = ds.cell_faces.p;
}


int upload_reference(DistanceState& ds, int64_t V, const float* xyz, int64_t F, const int32_t* faces, std::string& error, cudaStream_t st)
{
    if (V <= 0 || F <= 0) { error = format("the reference mesh needs V > 0 and F > 0, got V = %lld, F = %lld", static_cast<long long>(V), static_cast<long long>(F)); return 1; }
    if (!xyz || !faces) { error = "xyz or faces is NULL"; return 1; }
    if (V > INT_MAX || F > INT_MAX / 3)
    {
        error = format("%lld vertices and %lld faces exceed the int32 indices of a mesh", static_cast<long long>(V), static_cast<long long>(F));
        return 1;
    }
    for (int64_t i = 0; i < 3 * V; ++i)
        if (!std::isfinite(xyz[i])) { error = format("coordinate %lld of vertex %lld is not finite", static_cast<long long>(i % 3), static_cast<long long>(i / 3)); return 1; }
    for (int64_t i = 0; i < 3 * F; ++i)
        if (faces[i] < 0 || faces[i] >= V)
        {
            error = format("face %lld has vertex index %d outside [0, %lld)", static_cast<long long>(i / 3), faces[i], static_cast<long long>(V));
            return 1;
        }
    ds.have_ref = false;
    ds.ref_vpos.ensure(3 * static_cast<size_t>(V)); ds.ref_faces.ensure(static_cast<size_t>(F));
    CK(cudaMemcpyAsync(ds.ref_vpos.p, xyz, 3 * static_cast<size_t>(V) * sizeof(float), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ds.ref_faces.p, faces, static_cast<size_t>(F) * sizeof(int3), cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
    ds.ref_V = V; ds.ref_F = F; ds.have_ref = true;
    return 0;
}

int compute(DistanceState& ds, const DistMesh& a, const I3DDistanceParams& p, I3DDistanceInfo* info, std::string& error, cudaStream_t st)
{
    if (!ds.ev_ready) { for (auto& ev : ds.ev) CK(cudaEventCreate(&ev)); ds.ev_ready = true; }
    const DistMesh b{ds.ref_V, ds.ref_F, ds.ref_vpos.p, ds.ref_faces.p};
    // both grids are sized, and refused, before anything is written
    DistGrid gb, ga;
    int64_t eb = 0, ea = 0;
    if (!plan(ds.grid, b, p.cell_size, p.max_distance, gb, eb, nullptr, error, st) || !plan(ds.grid, a, p.cell_size, p.max_distance, ga, ea, nullptr, error, st))
        return 1;
    const int L = p.samples_per_edge, LL = L * L;
    DistQuery q;
    std::memset(&q, 0, sizeof(q));
    q.max_distance = p.max_distance; q.L = L; q.num_thresholds = p.num_thresholds;
    for (int k = 0; k < p.num_thresholds; ++k) q.tau[k] = p.thresholds[k];
    const DistMesh src[2] = {a, b};
    DistGrid* grid[2] = {&gb, &ga};
    const DistMesh* tgt[2] = {&b, &a};
    const int64_t ns[2] = {a.F * LL, b.F * LL};
    const unsigned nbs[2] = {blocks_for(static_cast<size_t>(ns[0])), blocks_for(static_cast<size_t>(ns[1]))};
    ds.partials.ensure(static_cast<size_t>(std::max(nbs[0], nbs[1])) * kDistStats);
    ds.stats.ensure(2 * kDistStats);
    ds.vdist.ensure(static_cast<size_t>(a.V)); ds.vface.ensure(static_cast<size_t>(a.V));
    ds.have_keep = false;
    for (int d = 0; d < 2; ++d)
    {
        if (ds.keep) { ds.keep_d2[d].ensure(static_cast<size_t>(ns[d])); ds.keep_face[d].ensure(static_cast<size_t>(ns[d])); }
        ds.keep_n[d] = ds.keep ? ns[d] : 0;
    }
    ds.vtests.ensure(1);
    CK(cudaMemsetAsync(ds.vtests.p, 0, sizeof(unsigned long long), st));
    for (int d = 0; d < 2; ++d)
    {
        cudaEvent_t* ev = ds.ev + (d == 0 ? 0 : 8);
        CK(cudaEventRecord(ev[0], st));
        build(ds.grid, *tgt[d], *grid[d], d == 0 ? eb : ea, st);
        CK(cudaEventRecord(ev[1], st));
        k_dist_samples<<<nbs[d], kThreads, 0, st>>>(src[d], *tgt[d], *grid[d], q, ds.keep ? ds.keep_d2[d].p : nullptr, ds.keep ? ds.keep_face[d].p : nullptr,
                                                    ds.partials.p);
        CK(cudaEventRecord(ev[2], st));
        k_dist_finish<<<1, 32 * kDistStats, 0, st>>>(static_cast<int>(nbs[d]), ds.partials.p, ds.stats.p + d * kDistStats);
        CK(cudaEventRecord(ev[3], st));
        if (d == 0)
        {
            CK(cudaEventRecord(ds.ev[4], st));
            k_dist_vertices<<<blocks_for(static_cast<size_t>(a.V)), kThreads, 0, st>>>(a, b, gb, p.max_distance, ds.vdist.p, ds.vface.p, ds.vtests.p);
            CK(cudaEventRecord(ds.ev[5], st));
        }
    }
    double s[2 * kDistStats];
    unsigned long long vt = 0;
    CK(cudaMemcpyAsync(s, ds.stats.p, sizeof(s), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&vt, ds.vtests.p, sizeof(vt), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    ds.result_V = a.V; ds.have_result = true; ds.have_keep = ds.keep;
    if (info)
    {
        I3DDistanceInfo inf;
        std::memset(&inf, 0, sizeof(inf));
        auto ms = [&](int i, int j) { float m = 0.f; CK(cudaEventElapsedTime(&m, ds.ev[i], ds.ev[j])); return static_cast<double>(m); };
        for (int d = 0; d < 2; ++d)
        {
            I3DDistanceSide& o = inf.side[d];
            side_info(s + d * kDistStats, *grid[d], ns[d], d == 0 ? eb : ea, p.num_thresholds, o);
            const int e0 = d == 0 ? 0 : 8;
            o.ms_grid = ms(e0, e0 + 1); o.ms_query = ms(e0 + 1, e0 + 2); o.ms_reduce = ms(e0 + 2, e0 + 3);
        }
        inf.num_thresholds = p.num_thresholds;
        for (int k = 0; k < p.num_thresholds; ++k)
        {
            const double P = inf.side[0].fraction[k], R = inf.side[1].fraction[k];
            inf.precision[k] = P; inf.recall[k] = R;
            inf.fscore[k] = P + R > 0.0 ? 2.0 * P * R / (P + R) : 0.0;
        }
        inf.num_vertices = a.V;
        inf.vertex_point_triangle_tests = static_cast<int64_t>(vt);
        inf.ms_vertices = ms(4, 5);
        *info = inf;
    }
    return 0;
}

bool check_rigid(const double* T, std::string& error)
{
    for (int i = 0; i < 12; ++i)
        if (!std::isfinite(T[i])) { error = format("entry %d of the transform is not finite", i); return false; }
    double dev = 0.0;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
        {
            const double d = T[i] * T[j] + T[3 + i] * T[3 + j] + T[6 + i] * T[6 + j] - (i == j ? 1.0 : 0.0);
            dev = std::max(dev, std::fabs(d));
        }
    const double det = T[0] * (T[4] * T[8] - T[5] * T[7]) - T[1] * (T[3] * T[8] - T[5] * T[6]) + T[2] * (T[3] * T[7] - T[4] * T[6]);
    if (dev > 1e-5 || det < 0.0)
    {
        error = format("the transform's R is not a rotation (max |R^T R - I| = %g, det R = %g)", dev, det);
        return false;
    }
    return true;
}

int register_reference(DistanceState& ds, const DistMesh& a, const I3DRegisterParams& p, const double* T_init, double* T_out, I3DRegisterInfo* info,
                       std::string& error, cudaStream_t st)
{
    const DistMesh b{ds.ref_V, ds.ref_F, ds.ref_vpos.p, ds.ref_faces.p};
    DistGrid g;
    int64_t entries = 0;
    if (!plan(ds.grid, b, p.cell_size, p.max_distance[0], g, entries, nullptr, error, st)) return 1;
    int E = 1;                                   // every system: one per update, then the one at the final pose
    for (int s = 0; s < p.num_stages; ++s) E += p.iterations[s];
    const int L = p.samples_per_edge;
    const int64_t ns = a.F * L * L;
    const unsigned nb = blocks_for(static_cast<size_t>(ns));
    ds.reg_state.ensure(1); ds.reg_T.ensure(12); ds.reg_partials.ensure(static_cast<size_t>(nb) * kTrackVals); ds.reg_wpartials.ensure(2 * static_cast<size_t>(nb));
    ds.reg_sums.ensure(static_cast<size_t>(E) * kTrackVals); ds.reg_sys.ensure(kTrackVals); ds.reg_poses.ensure(12 * static_cast<size_t>(E));
    ds.reg_face.ensure(static_cast<size_t>(ns)); ds.reg_counters.ensure(2);
    const size_t nev = 2 + 3 * static_cast<size_t>(E);
    while (ds.reg_ev.size() < nev) { cudaEvent_t ev; CK(cudaEventCreate(&ev)); ds.reg_ev.push_back(ev); }
    static const double kIdentity[12] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0};
    ds.have_reg = false;
    CK(cudaMemcpyAsync(ds.reg_T.p, T_init ? T_init : kIdentity, 12 * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(ds.reg_counters.p, 0, 2 * sizeof(unsigned long long), st));
    cudaEvent_t* ev = ds.reg_ev.data();
    CK(cudaEventRecord(ev[0], st));
    build(ds.grid, b, g, entries, st);
    CK(cudaEventRecord(ev[1], st));
    track::pose_init(ds.reg_T.p, ds.reg_state.p, st);
    int e = 0;
    auto system = [&](float max_distance, int solve) {
        const RegQuery q{L, max_distance, p.min_normal_cos, p.min_normal_cos > -1.0f ? 1 : 0};
        // the pose M (TrackState::T) this system is formed at
        CK(cudaMemcpyAsync(ds.reg_poses.p + 12 * static_cast<size_t>(e), ds.reg_state.p, 12 * sizeof(double), cudaMemcpyDeviceToDevice, st));
        double* wp = e == 0 ? ds.reg_wpartials.p : (e == E - 1 ? ds.reg_wpartials.p + nb : nullptr);
        CK(cudaEventRecord(ev[2 + 3 * e], st));
        k_reg_rows<<<nb, kThreads, 0, st>>>(a, b, g, q, ds.reg_state.p, e == 0 ? ds.reg_face.p : nullptr, ds.reg_partials.p, wp, ds.reg_counters.p);
        CK(cudaEventRecord(ev[3 + 3 * e], st));
        track::pose_step(static_cast<int>(nb), ds.reg_partials.p, ds.reg_sums.p + static_cast<size_t>(e) * kTrackVals, ds.reg_state.p, ds.reg_sys.p,
                         p.min_correspondences, solve, ds.reg_counters.p + 1, st);
        CK(cudaEventRecord(ev[4 + 3 * e], st));
        ++e;
    };
    for (int s = 0; s < p.num_stages; ++s)
        for (int it = 0; it < p.iterations[s]; ++it) system(p.max_distance[s], 1);
    system(p.max_distance[p.num_stages - 1], 0);
    TrackState hs;
    std::vector<double> sums(static_cast<size_t>(E) * kTrackVals), wp(2 * static_cast<size_t>(nb));
    unsigned long long counters[2] = {0, 0};
    CK(cudaMemcpyAsync(&hs, ds.reg_state.p, sizeof(hs), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(sums.data(), ds.reg_sums.p, sums.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(wp.data(), ds.reg_wpartials.p, wp.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(counters, ds.reg_counters.p, sizeof(counters), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    // sum w of the first and the last system: the blocks in order, as k_tile_sums adds them
    for (int k = 0; k < 2; ++k)
    {
        const double* w = wp.data() + (E == 1 ? 0 : k) * static_cast<size_t>(nb);
        double s = 0.0;
        for (unsigned i = 0; i < nb; ++i) s += w[i];
        ds.reg_wsum[k] = s;
    }
    ds.reg_n = E; ds.reg_samples = ns; ds.have_reg = true;
    std::memcpy(T_out, hs.w2c, 12 * sizeof(double));
    if (info)
    {
        I3DRegisterInfo inf;
        std::memset(&inf, 0, sizeof(inf));
        inf.status = hs.status; inf.iterations = hs.iterations; inf.update_norm = hs.update_norm;
        const double* S0 = sums.data();
        const double* S1 = sums.data() + static_cast<size_t>(E - 1) * kTrackVals;
        inf.initial_rows = static_cast<int64_t>(S0[28]); inf.final_rows = static_cast<int64_t>(S1[28]);
        inf.initial_weight = ds.reg_wsum[0]; inf.final_weight = ds.reg_wsum[1];
        inf.initial_residual_sq = S0[27]; inf.final_residual_sq = S1[27];
        inf.initial_rms = inf.initial_weight > 0.0 ? std::sqrt(S0[27] / inf.initial_weight) : 0.0;
        inf.final_rms = inf.final_weight > 0.0 ? std::sqrt(S1[27] / inf.final_weight) : 0.0;
        inf.num_samples = ns;
        inf.point_triangle_tests = static_cast<int64_t>(counters[0]);
        inf.cell_size = g.h;
        for (int k = 0; k < 3; ++k) inf.grid[k] = g.n[k];
        inf.num_cells = static_cast<int64_t>(g.n[0]) * g.n[1] * g.n[2];
        inf.num_cell_entries = entries;
        auto ms = [&](int i, int j) { float m = 0.f; CK(cudaEventElapsedTime(&m, ev[i], ev[j])); return static_cast<double>(m); };
        inf.ms_grid = ms(0, 1);
        for (int k = 0; k < E; ++k) { inf.ms_rows += ms(2 + 3 * k, 3 + 3 * k); inf.ms_solve += ms(3 + 3 * k, 4 + 3 * k); }
        *info = inf;
    }
    return 0;
}

void transform_reference(DistanceState& ds, const double* T, cudaStream_t st)
{
    ds.reg_T.ensure(12);
    CK(cudaMemcpyAsync(ds.reg_T.p, T, 12 * sizeof(double), cudaMemcpyHostToDevice, st));
    k_reg_transform<<<blocks_for(static_cast<size_t>(ds.ref_V)), kThreads, 0, st>>>(ds.ref_V, ds.ref_vpos.p, ds.reg_T.p);
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
}

} // namespace distance
} // namespace i3d
