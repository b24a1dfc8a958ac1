// fusion_oracle.cpp — float CPU restatement of the reference's RGB-D fusion chain (AppFusion::fuseSDF,
// apps/src/app_fusion.cpp:107-200; paths below relative to libintrinsic3d/).  The checker of intrinsic3d_b200/csrc/i3d_fusion.cuh:
// plain serial loops over a std::unordered_map grid, as the reference runs them, one float operation at a time
// (built with -ffp-contract=off), vector sums left to right like the engine.  Not part of the product.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <unordered_map>
#include <vector>

namespace
{
struct Cam { int W, H; float fx, fy, cx, cy; };
struct Params
{
    float voxel_size, depth_min, depth_max, weight_sample;
    float clip[6];
    int window, iterations;
};
struct Voxel { float sdf = 0.0f; float weight = 0.0f; uint8_t c[3] = {0, 0, 0}; };     // sparse_voxel_grid.h:56-62

uint64_t pack(int x, int y, int z)
{
    return ((static_cast<uint64_t>(x + (1 << 20)) & 0x1FFFFFull) << 42) | ((static_cast<uint64_t>(y + (1 << 20)) & 0x1FFFFFull) << 21) |
           (static_cast<uint64_t>(z + (1 << 20)) & 0x1FFFFFull);
}
uint64_t order_key(int x, int y, int z)
{
    const uint64_t ux = static_cast<uint64_t>(x + (1 << 20)), uy = static_cast<uint64_t>(y + (1 << 20)), uz = static_cast<uint64_t>(z + (1 << 20));
    return ((uz >> 3) << 46) | ((uy >> 3) << 28) | ((ux >> 3) << 10) | ((uz & 7ull) << 6) | ((uy & 7ull) << 3) | (ux & 7ull);
}
// (int) cast, saturating where C++ leaves it undefined
int f2i(float v)
{
    if (!(v == v)) return 0;
    if (v >= 2147483648.0f) return INT_MAX;
    if (v < -2147483648.0f) return INT_MIN;
    return static_cast<int>(v);
}
// SparseVoxelGrid::worldToVoxel = nv::round(p * (1 / voxel_size)) (sparse_voxel_grid.cpp:211-220, include/nv/mat.h:90)
int w2v(float p, float inv) { return f2i(p * inv + 0.5f); }
void xform(const float* R, const float* t, const float p[3], float q[3])
{
    for (int k = 0; k < 3; ++k)
    {
        float s = R[3 * k] * p[0];
        s = s + R[3 * k + 1] * p[1];
        s = s + R[3 * k + 2] * p[2];
        q[k] = s + t[k];
    }
}
bool in_bounds(const int b[6], int x, int y, int z) { return !(x < b[0] || x > b[1] || y < b[2] || y > b[3] || z < b[4] || z > b[5]); }
// math::robustKernel(val, 2) (src/math.cpp:43-47)
float robust(float v) { const float div = 1.0f + 2.0f * v; return 1.0f / (div * div * div); }
float norm3(float a, float b, float c) { return std::sqrt((a * a + b * b) + c * c); }

struct Fusion
{
    Params P;
    float trunc, step, inv;
    bool use_clip;
    std::unordered_map<uint64_t, Voxel> grid;
    std::vector<int> cx, cy, cz;          // coordinates by insertion, for iteration

    explicit Fusion(const Params& p) : P(p)
    {
        trunc = P.voxel_size * 5.0f; step = P.voxel_size * 0.25f; inv = 1.0f / P.voxel_size;        // sparse_voxel_grid.cpp:48, :403
        float sq = 0.0f;
        for (int k = 0; k < 6; ++k) sq += P.clip[k] * P.clip[k];
        use_clip = sq > 0.0f;
    }
    void add(int x, int y, int z)
    {
        const uint64_t k = pack(x, y, z);
        if (grid.find(k) != grid.end()) return;
        grid.emplace(k, Voxel());
        cx.push_back(x); cy.push_back(y); cz.push_back(z);
    }
};

// erodeDiscontinuities (src/rgbd/processing.cpp:184-235)
void erode(int W, int H, int window, const float* in, float* out)
{
    if (window <= 0) { std::memcpy(out, in, sizeof(float) * W * H); return; }
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x)
        {
            const float d_ref = in[y * W + x];
            if (d_ref == 0.0f) { out[y * W + x] = 0.0f; continue; }
            bool valid = true;
            for (int v = std::max(0, y - window); v <= std::min(y + window, H - 1) && valid; ++v)
                for (int u = std::max(0, x - window); u <= std::min(x + window, W - 1); ++u)
                {
                    const float d = in[v * W + u];
                    if (d == 0.0f || std::fabs(d - d_ref) > 0.5f) { valid = false; break; }
                }
            out[y * W + x] = valid ? d_ref : 0.0f;
        }
}

// computeVertexMap + computeNormals(vertex_map, 0.3) (processing.cpp:49-126)
void normals(const Cam& c, const float* depth, float* n)
{
    const int W = c.W, H = c.H;
    const float fxi = 1.0f / c.fx, fyi = 1.0f / c.fy;
    std::vector<float> vm(3 * static_cast<size_t>(W) * H);
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x)
        {
            const float d = depth[y * W + x];
            const float x0 = (static_cast<float>(x) - c.cx) * fxi, y0 = (static_cast<float>(y) - c.cy) * fyi;
            float* v = &vm[3 * (static_cast<size_t>(y) * W + x)];
            v[0] = x0 * d; v[1] = y0 * d; v[2] = d;
        }
    std::memset(n, 0, sizeof(float) * 3 * W * H);
    for (int y = 1; y < H - 1; ++y)
        for (int x = 1; x < W - 1; ++x)
        {
            const float* v = &vm[3 * (static_cast<size_t>(y) * W + x)];
            if (v[2] == 0.0f) continue;
            const float* x0 = &vm[3 * (static_cast<size_t>(y) * W + x - 1)];
            const float* x1 = &vm[3 * (static_cast<size_t>(y) * W + x + 1)];
            const float* y0 = &vm[3 * (static_cast<size_t>(y - 1) * W + x)];
            const float* y1 = &vm[3 * (static_cast<size_t>(y + 1) * W + x)];
            if (x0[2] == 0.0f || x1[2] == 0.0f || y0[2] == 0.0f || y1[2] == 0.0f) continue;
            const float tx[3] = {x1[0] - x0[0], x1[1] - x0[1], x1[2] - x0[2]};
            const float ty[3] = {y1[0] - y0[0], y1[1] - y0[1], y1[2] - y0[2]};
            if (norm3(tx[0], tx[1], tx[2]) < 0.3f && norm3(ty[0], ty[1], ty[2]) < 0.3f)
            {
                float cr[3] = {ty[1] * tx[2] - ty[2] * tx[1], ty[2] * tx[0] - ty[0] * tx[2], ty[0] * tx[1] - ty[1] * tx[0]};
                const float sq = (cr[0] * cr[0] + cr[1] * cr[1]) + cr[2] * cr[2];
                if (sq > 0.0f) { const float l = std::sqrt(sq); cr[0] = cr[0] / l; cr[1] = cr[1] / l; cr[2] = cr[2] / l; }
                float* o = &n[3 * (static_cast<size_t>(y) * W + x)];
                o[0] = cr[0]; o[1] = cr[1]; o[2] = cr[2];
            }
        }
}

// computeFrustumBounds (sparse_voxel_grid.cpp:572-602) + computeFrustumPoints (src/math.cpp:131-148)
void bounds(const Cam& cam, float dmin, float dmax, float vs, const float* R, const float* t, int b[6])
{
    const float inv = 1.0f / vs;
    const int px[4] = {0, cam.W - 1, cam.W - 1, 0}, py[4] = {0, 0, cam.H - 1, cam.H - 1};
    b[0] = b[2] = b[4] = INT_MAX; b[1] = b[3] = b[5] = INT_MIN;
    for (int i = 0; i < 8; ++i)
    {
        const float d = i < 4 ? dmin : dmax;
        float c[3] = {0.0f, 0.0f, 0.0f};
        if (d != 0.0f)
        {
            const float x = (static_cast<float>(px[i & 3]) - cam.cx) / cam.fx, y = (static_cast<float>(py[i & 3]) - cam.cy) / cam.fy;
            c[0] = d * x; c[1] = d * y; c[2] = d;
        }
        float p[3];
        xform(R, t, c, p);
        for (int k = 0; k < 3; ++k)
        {
            const int pl = w2v(static_cast<float>(f2i(std::floor(p[k]))), inv), pu = w2v(static_cast<float>(f2i(std::ceil(p[k]))), inv);
            b[2 * k] = std::min(b[2 * k], std::min(pl, pu));
            b[2 * k + 1] = std::max(b[2 * k + 1], std::max(pl, pu));
        }
    }
}

// SparseVoxelGrid::alloc (sparse_voxel_grid.cpp:398-467).  Returns 2 when a voxel to allocate is outside pack()'s range.
int alloc(Fusion& fu, const Cam& cam, const float* depth, const float* R, const float* t, const int b[6])
{
    const int lim = (1 << 20) - 2;
    for (int y = 0; y < cam.H; ++y)
        for (int x = 0; x < cam.W; ++x)
        {
            const float d = depth[y * cam.W + x];
            if (d == 0.0f) continue;
            const float pc[3] = {(static_cast<float>(x) - cam.cx) / cam.fx, (static_cast<float>(y) - cam.cy) / cam.fy, 1.0f};   // unproject2(x, y, 1)
            int last[3] = {0, 0, 0};
            for (float d_off = -fu.trunc; d_off <= fu.trunc; d_off += fu.step)
            {
                const float s = d + d_off;
                const float pr[3] = {pc[0] * s, pc[1] * s, pc[2] * s};
                float pw[3];
                xform(R, t, pr, pw);
                const int g[3] = {w2v(pw[0], fu.inv), w2v(pw[1], fu.inv), w2v(pw[2], fu.inv)};
                if (g[0] == last[0] && g[1] == last[1] && g[2] == last[2]) continue;
                last[0] = g[0]; last[1] = g[1]; last[2] = g[2];
                if (!in_bounds(b, g[0], g[1], g[2])) continue;
                if (fu.use_clip)
                {
                    const float w0 = static_cast<float>(g[0]) * fu.P.voxel_size, w1 = static_cast<float>(g[1]) * fu.P.voxel_size,
                                w2 = static_cast<float>(g[2]) * fu.P.voxel_size;
                    if (w0 < fu.P.clip[0] || w0 > fu.P.clip[1] || w1 < fu.P.clip[2] || w1 > fu.P.clip[3] || w2 < fu.P.clip[4] || w2 > fu.P.clip[5]) continue;
                }
                if (std::abs(g[0]) > lim || std::abs(g[1]) > lim || std::abs(g[2]) > lim) return 2;
                for (int dz = -1; dz <= 1; ++dz)
                    for (int dy = -1; dy <= 1; ++dy)
                        for (int dx = -1; dx <= 1; ++dx) fu.add(g[0] + dx, g[1] + dy, g[2] + dz);
            }
        }
    return 0;
}

// SparseVoxelGrid::integrate's per-voxel update (sparse_voxel_grid.cpp:316-392)
void integrate(Fusion& fu, const Cam& dc, const Cam& cc, const float* depth, const float* nrm, const uint8_t* bgr, const float* R, const float* t,
               const int b[6])
{
    const Params& P = fu.P;
    for (size_t i = 0; i < fu.cx.size(); ++i)
    {
        const int X = fu.cx[i], Y = fu.cy[i], Z = fu.cz[i];
        if (!in_bounds(b, X, Y, Z)) continue;
        Voxel& v = fu.grid[pack(X, Y, Z)];
        const float pw[3] = {static_cast<float>(X) * P.voxel_size, static_cast<float>(Y) * P.voxel_size, static_cast<float>(Z) * P.voxel_size};
        float p[3];
        xform(R, t, pw, p);
        if (p[2] < 0.0f) continue;
        const int u = f2i(((p[0] * dc.fx) / p[2] + dc.cx) + 0.5f), vv = f2i(((p[1] * dc.fy) / p[2] + dc.cy) + 0.5f);
        if (u < 0 || vv < 0 || u >= dc.W || vv >= dc.H) continue;
        const size_t pix = static_cast<size_t>(vv) * dc.W + u;
        const float d = depth[pix];
        if (d <= 0.0f) continue;
        const float sdf = d - p[2];
        if (sdf <= -fu.trunc) continue;
        const float tsdf = sdf >= 0.0f ? std::min(fu.trunc, sdf) : std::max(-fu.trunc, sdf);
        float wu = 1.0f;
        if (P.weight_sample > 0.0f)
        {
            float q[3] = {p[0], p[1], p[2]};
            const float sq = (q[0] * q[0] + q[1] * q[1]) + q[2] * q[2];
            if (sq > 0.0f) { const float l = std::sqrt(sq); q[0] = q[0] / l; q[1] = q[1] / l; q[2] = q[2] / l; }
            const float* n = nrm + 3 * pix;
            float w_normal = 1.0f - std::fabs((q[0] * n[0] + q[1] * n[1]) + q[2] * n[2]);
            w_normal = std::max(std::min(w_normal, 1.0f), 0.0f);
            w_normal = std::max(P.weight_sample * robust(w_normal), 1.0f);
            const float w_dist = std::max(P.weight_sample * robust((2.0f * std::fabs(tsdf)) / fu.trunc), 1.0f);
            const float d_norm = (d - P.depth_min) / (P.depth_max - P.depth_min);
            const float w_depth = std::max(P.weight_sample * (1.0f - d_norm), 1.0f);
            wu = std::max(((w_normal + w_dist) + w_depth) / 3.0f, 3.0f);
        }
        const float w_old = v.weight, w_new = w_old + wu;
        v.sdf = (v.sdf * w_old + sdf * wu) / w_new;                 // unclamped sdf
        const int cu = f2i(((p[0] * cc.fx) / p[2] + cc.cx) + 0.5f), cv = f2i(((p[1] * cc.fy) / p[2] + cc.cy) + 0.5f);
        if (cu >= 0 && cv >= 0 && cu < cc.W && cv < cc.H)
        {
            const uint8_t* px = bgr + (static_cast<size_t>(cv) * cc.W + cu) * 3;
            const float cn[3] = {static_cast<float>(px[2]), static_cast<float>(px[1]), static_cast<float>(px[0])};
            for (int k = 0; k < 3; ++k) v.c[k] = static_cast<uint8_t>(f2i((static_cast<float>(v.c[k]) * w_old + cn[k] * wu) / w_new));
        }
        v.weight = w_new;
    }
}

std::vector<int> canonical(const Fusion& fu, bool valid_only)
{
    std::vector<std::pair<uint64_t, int>> k;
    for (size_t i = 0; i < fu.cx.size(); ++i)
    {
        if (valid_only && !(fu.grid.at(pack(fu.cx[i], fu.cy[i], fu.cz[i])).weight > 0.0f)) continue;
        k.emplace_back(order_key(fu.cx[i], fu.cy[i], fu.cz[i]), static_cast<int>(i));
    }
    std::sort(k.begin(), k.end());
    std::vector<int> out;
    for (auto& e : k) out.push_back(e.second);
    return out;
}

// SDFAlgorithms::correctSDF (src/sdf/algorithms.cpp:260-337) in canonical order.  jacobi: neighbours from the previous sweep (the
// device schedule); otherwise in place (Gauss-Seidel, the reference's schedule in its iteration order).  Returns the sweeps run.
int correct(Fusion& fu, bool jacobi)
{
    const std::vector<int> ord = canonical(fu, false);
    const size_t n = ord.size();
    std::vector<float> s(n), w(n);
    std::unordered_map<uint64_t, int> at;
    for (size_t i = 0; i < n; ++i)
    {
        const Voxel& v = fu.grid.at(pack(fu.cx[ord[i]], fu.cy[ord[i]], fu.cz[ord[i]]));
        s[i] = v.sdf; w[i] = v.weight;
        at.emplace(pack(fu.cx[ord[i]], fu.cy[ord[i]], fu.cz[ord[i]]), static_cast<int>(i));
    }
    const float vs = fu.P.voxel_size;
    int sweeps = 0;
    for (int it = 0; it < fu.P.iterations; ++it)
    {
        ++sweeps;
        bool has_update = false;
        std::vector<float> s2 = s, w2 = w;
        std::vector<float>& so = jacobi ? s2 : s;
        std::vector<float>& wo = jacobi ? w2 : w;
        for (size_t i = 0; i < n; ++i)
        {
            if (!(w[i] > 0.0f)) continue;                   // valid(); validity never changes (updates set weight 1)
            const int x = fu.cx[ord[i]], y = fu.cy[ord[i]], z = fu.cz[ord[i]];
            const double sdf = static_cast<double>(s[i]);   // sweep-start value (in place: the value this voxel has now)
            const double sgn = sdf >= 0.0 ? 1.0 : -1.0;
            const float cx = static_cast<float>(x) * vs, cy = static_cast<float>(y) * vs, cz = static_cast<float>(z) * vs;
            for (int k = -1; k <= 1; ++k)
                for (int j = -1; j <= 1; ++j)
                    for (int ii = -1; ii <= 1; ++ii)
                    {
                        if (k == 0 && j == 0 && ii == 0) continue;
                        auto f = at.find(pack(x + ii, y + j, z + k));
                        if (f == at.end() || !(w[f->second] > 0.0f)) continue;
                        const double sdf_nb = static_cast<double>(s[f->second]);
                        const double sgn_nb = sdf_nb >= 0.0 ? 1.0 : -1.0;
                        const float dx = cx - static_cast<float>(x + ii) * vs, dy = cy - static_cast<float>(y + j) * vs, dz = cz - static_cast<float>(z + k) * vs;
                        const double dist_nb = sdf_nb + sgn_nb * static_cast<double>(norm3(dx, dy, dz));
                        if (std::fabs(dist_nb) < std::fabs(sdf) && sgn == sgn_nb)
                        {
                            so[i] = static_cast<float>(dist_nb);
                            wo[i] = 1.0f;
                            has_update = true;
                        }
                    }
        }
        if (jacobi) { s.swap(s2); w.swap(w2); }
        if (!has_update) break;
    }
    for (size_t i = 0; i < n; ++i)
    {
        Voxel& v = fu.grid.at(pack(fu.cx[ord[i]], fu.cy[ord[i]], fu.cz[ord[i]]));
        v.sdf = s[i]; v.weight = w[i];
    }
    return sweeps;
}
} // namespace

extern "C" {

void* fo_create(const float* pf /* voxel_size, depth_min, depth_max, weight_sample, clip[6] */, int window, int iterations)
{
    Params p;
    p.voxel_size = pf[0]; p.depth_min = pf[1]; p.depth_max = pf[2]; p.weight_sample = pf[3];
    for (int k = 0; k < 6; ++k) p.clip[k] = pf[4 + k];
    p.window = window; p.iterations = iterations;
    return new Fusion(p);
}
void* fo_clone(void* h) { return new Fusion(*static_cast<Fusion*>(h)); }
void fo_destroy(void* h) { delete static_cast<Fusion*>(h); }

void fo_erode(int W, int H, int window, const float* in, float* out) { erode(W, H, window, in, out); }
void fo_normals(const int* wh, const float* k4, const float* depth, float* n) { normals(Cam{wh[0], wh[1], k4[0], k4[1], k4[2], k4[3]}, depth, n); }
void fo_bounds(const int* wh, const float* k4, float dmin, float dmax, float vs, const float* Rt, int* b)
{
    bounds(Cam{wh[0], wh[1], k4[0], k4[1], k4[2], k4[3]}, dmin, dmax, vs, Rt, Rt + 9, b);
}

// fuses F frames; returns 0, or 2 when a voxel lies outside the packable range
int fo_integrate(void* h, int F, const int* dwh, const float* dk, const float* depth, const int* cwh, const float* ck, const uint8_t* bgr,
                 const float* c2w, const float* w2c)
{
    Fusion& fu = *static_cast<Fusion*>(h);
    const Cam dc{dwh[0], dwh[1], dk[0], dk[1], dk[2], dk[3]}, cc{cwh[0], cwh[1], ck[0], ck[1], ck[2], ck[3]};
    const size_t dimg = static_cast<size_t>(dc.W) * dc.H, cimg = static_cast<size_t>(cc.W) * cc.H * 3;
    std::vector<float> d(dimg), n(3 * dimg);
    for (int f = 0; f < F; ++f)
    {
        erode(dc.W, dc.H, fu.P.window, depth + dimg * f, d.data());
        if (fu.P.weight_sample > 0.0f) normals(dc, d.data(), n.data());
        int b[6];
        bounds(dc, fu.P.depth_min, fu.P.depth_max, fu.P.voxel_size, c2w + 12 * f, c2w + 12 * f + 9, b);
        if (alloc(fu, dc, d.data(), c2w + 12 * f, c2w + 12 * f + 9, b)) return 2;
        integrate(fu, dc, cc, d.data(), n.data(), bgr + cimg * f, w2c + 12 * f, w2c + 12 * f + 9, b);
    }
    return 0;
}

// correctSDF (mode 1 Jacobi, 2 Gauss-Seidel, 0 none) then clearInvalidVoxels; returns the sweeps run
int fo_finish(void* h, int mode)
{
    Fusion& fu = *static_cast<Fusion*>(h);
    const int sweeps = mode ? correct(fu, mode == 1) : 0;
    Fusion kept(fu.P);
    for (int i : canonical(fu, true))
    {
        kept.add(fu.cx[i], fu.cy[i], fu.cz[i]);
        kept.grid[pack(fu.cx[i], fu.cy[i], fu.cz[i])] = fu.grid.at(pack(fu.cx[i], fu.cy[i], fu.cz[i]));
    }
    fu = kept;
    return sweeps;
}

int64_t fo_num(void* h) { return static_cast<int64_t>(static_cast<Fusion*>(h)->cx.size()); }

// the volume in canonical order
void fo_volume(void* h, int32_t* xyz, float* sdf, float* w, uint8_t* rgb)
{
    Fusion& fu = *static_cast<Fusion*>(h);
    const std::vector<int> ord = canonical(fu, false);
    for (size_t i = 0; i < ord.size(); ++i)
    {
        const int j = ord[i];
        const Voxel& v = fu.grid.at(pack(fu.cx[j], fu.cy[j], fu.cz[j]));
        xyz[3 * i] = fu.cx[j]; xyz[3 * i + 1] = fu.cy[j]; xyz[3 * i + 2] = fu.cz[j];
        sdf[i] = v.sdf; w[i] = v.weight;
        rgb[3 * i] = v.c[0]; rgb[3 * i + 1] = v.c[1]; rgb[3 * i + 2] = v.c[2];
    }
}

} // extern "C"
