/*
 * i3d_lighting.cuh — SVSH lighting on the device (SURVEY.md §8 a15 / f1).
 *
 * Replaces LightingSVSH::estimate + computeVoxelShCoeffs
 * (libintrinsic3d/src/lighting/lighting_svsh.cpp:93-110,166-346) and Subvolumes
 * (src/lighting/subvolumes.cpp:66-304):
 *
 *   k_svsh_bounds / k_svsh_mark / k_svsh_number / k_svsh_indices / k_svsh_neighbors
 *       Subvolumes::generate: occupied cubes floor(p / size) of ALL hash voxels, numbered in ascending
 *       (z, y, x) order through a dense table over their bounding box.
 *   k_svsh_accumulate
 *       one SHDataCost row per contributing voxel (row = albedo * basis(n), target lum/255, weight
 *       sdfToWeight).  The rows of a subvolume touch only its 9 unknowns, so instead of storing N_a x 9
 *       rows the kernel accumulates the per-subvolume normal equations H_s = sum w j j^T (45), g_s = sum w l j
 *       (9), c_s = sum w l^2 and sum w in float64: one pass over the voxels, warp-level reduction per
 *       distinct subvolume, 57 double atomics per (warp, subvolume).
 *   k_svsh_solve
 *       the whole ceres::Solve (trust-region LM, CGNR with the 9x9 block-Jacobi preconditioner, Jacobi
 *       column scaling, Q-based CG termination, function/gradient/parameter tolerances) on the reduced
 *       9S-unknown system in ONE single-CTA launch: J^T J = blockdiag(H_s) + (2 lambda / P) * graph
 *       Laplacian of the subvolume ring adjacency; CGNR on J and CG on J^T J are the same iteration.
 *       The problem is linear, so cost, gradient and model change are exact functions of (H, g, c).
 *   k_svsh_interpolate
 *       Subvolumes::interpolate(linear): trilinear blend of the 8 surrounding subvolume vectors at
 *       p / size - 0.5, missing cubes dropped and the weights renormalised (math::average).
 *
 * Float steps that decide an integer (cube index, corner cell) use exact-rounding intrinsics so that they
 * agree with the reference's float arithmetic (and oracle.cpp, compiled -ffp-contract=off).
 */
#pragma once
#include <limits.h>
#include "i3d_grid.cuh"
#include "../../include/i3d_types.h"

namespace i3d
{

constexpr int kLightAcc = 57;          // 45 (upper triangle of H) + 9 (g) + c + sum w + row count
constexpr int kLightSolveThreads = 1024;

// Subvolumes::pointToIndex of SparseVoxelGrid::voxelToWorld(v): floor((float(v) * voxel_size) * (1.0f / size))
__device__ __forceinline__ int sub_point_to_index(int v, float voxel_size, float inv_size)
{
    return static_cast<int>(floorf(FM(FM(static_cast<float>(v), voxel_size), inv_size)));
}

// bounds[0..2] = min index per axis, bounds[3..5] = max (initialised to INT_MAX / INT_MIN by the host)
__global__ void k_svsh_bounds(int64_t n, const int32_t* __restrict__ x, const int32_t* __restrict__ y, const int32_t* __restrict__ z, float voxel_size,
                              float inv_size, int* __restrict__ bounds)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
    if (i < n)
    {
        lo[0] = hi[0] = sub_point_to_index(x[i], voxel_size, inv_size);
        lo[1] = hi[1] = sub_point_to_index(y[i], voxel_size, inv_size);
        lo[2] = hi[2] = sub_point_to_index(z[i], voxel_size, inv_size);
    }
#pragma unroll
    for (int d = 0; d < 3; ++d)
    {
        lo[d] = __reduce_min_sync(0xffffffffu, lo[d]);
        hi[d] = __reduce_max_sync(0xffffffffu, hi[d]);
    }
    if ((threadIdx.x & 31) == 0)
    {
#pragma unroll
        for (int d = 0; d < 3; ++d) { atomicMin(&bounds[d], lo[d]); atomicMax(&bounds[3 + d], hi[d]); }
    }
}

__global__ void k_svsh_mark(int64_t n, const int32_t* __restrict__ x, const int32_t* __restrict__ y, const int32_t* __restrict__ z, float voxel_size,
                            SubvolGrid sg, int32_t* __restrict__ table)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    const int ix = sub_point_to_index(x[i], voxel_size, sg.inv_size) - sg.lo[0];
    const int iy = sub_point_to_index(y[i], voxel_size, sg.inv_size) - sg.lo[1];
    const int iz = sub_point_to_index(z[i], voxel_size, sg.inv_size) - sg.lo[2];
    table[(static_cast<int64_t>(iz) * sg.dim[1] + iy) * sg.dim[0] + ix] = 1;
}

// marks (0/1) -> ids in cell order (x fastest, then y, then z), -1 for empty cells.  One block.
__global__ void __launch_bounds__(kLightSolveThreads) k_svsh_number(int64_t cells, int32_t* __restrict__ table, int* __restrict__ count_out)
{
    __shared__ int s_cnt[kLightSolveThreads];
    const int tid = threadIdx.x;
    const int64_t chunk = (cells + kLightSolveThreads - 1) / kLightSolveThreads;
    const int64_t b = min(cells, tid * chunk), e = min(cells, b + chunk);
    int c = 0;
    for (int64_t i = b; i < e; ++i) c += table[i] != 0;
    s_cnt[tid] = c;
    __syncthreads();
    if (tid == 0)
    {
        int run = 0;
        for (int i = 0; i < kLightSolveThreads; ++i) { const int t = s_cnt[i]; s_cnt[i] = run; run += t; }
        *count_out = run;
    }
    __syncthreads();
    int id = s_cnt[tid];
    for (int64_t i = b; i < e; ++i) table[i] = table[i] != 0 ? id++ : -1;
}

// Subvolumes::index(i) for every id, and the ring neighbours (+x,-x,+y,-y,+z,-z; SDFAlgorithms::collectRingNeighborhood)
__global__ void k_svsh_indices(SubvolGrid sg, int32_t* __restrict__ sub_index /* [S][3] */, int32_t* __restrict__ sub_nbr /* [6][S] */, int S)
{
    const int64_t c = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (c >= sg.cells()) return;
    const int id = sg.table[c];
    if (id < 0) return;
    const int ix = static_cast<int>(c % sg.dim[0]);
    const int iy = static_cast<int>((c / sg.dim[0]) % sg.dim[1]);
    const int iz = static_cast<int>(c / (static_cast<int64_t>(sg.dim[0]) * sg.dim[1]));
    const int X = ix + sg.lo[0], Y = iy + sg.lo[1], Z = iz + sg.lo[2];
    sub_index[3 * id] = X; sub_index[3 * id + 1] = Y; sub_index[3 * id + 2] = Z;
    const int off[6][3] = {{1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};
#pragma unroll
    for (int d = 0; d < 6; ++d) sub_nbr[static_cast<int64_t>(d) * S + id] = sg.find(X + off[d][0], Y + off[d][1], Z + off[d][2]);
}

__device__ __forceinline__ double warp_allsum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// SHDataCost rows -> per-subvolume normal equations.  acc[S][kLightAcc], zeroed by the host.
__global__ void __launch_bounds__(kThreads) k_svsh_accumulate(GridView g, SubvolGrid sg, double thres_shell, int weighted, double* __restrict__ acc)
{
    const int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    const int lane = threadIdx.x & 31;
    int sid = -1;
    double vals[kLightAcc];
#pragma unroll
    for (int q = 0; q < kLightAcc; ++q) vals[q] = 0.0;
    if (v < g.n)
    {
        // lighting_svsh.cpp:203-228: valid, inside the thin shell, usable normal and albedo
        const double sdf = g.sdf[v];
        const double albedo = g.albedo[v];
        float nf[3];
        bool ok = g.weight[v] > 0.0f && !(fabs(sdf) > thres_shell);
        ok = ok && surface_normal_f(g, v, nf) && !(isnan(nf[0]) || isnan(nf[1]) || isnan(nf[2]));
        ok = ok && !(albedo == 0.0 || isnan(albedo));
        if (ok)
        {
            sid = sg.find(sub_point_to_index(g.x[v], g.voxel_size, sg.inv_size), sub_point_to_index(g.y[v], g.voxel_size, sg.inv_size),
                          sub_point_to_index(g.z[v], g.voxel_size, sg.inv_size));
            // Shading::shBasisFunctions<double> of the float normal (include/nv/shading.h:53-67)
            const double n0 = nf[0], n1 = nf[1], n2 = nf[2];
            double j[9];
            j[0] = 1.0; j[1] = n1; j[2] = n2; j[3] = n0; j[4] = n0 * n1; j[5] = n1 * n2;
            j[6] = (-n0 * n0) - (n1 * n1) + 2.0 * (n2 * n2); j[7] = n0 * n2; j[8] = (n0 * n0) - (n1 * n1);
#pragma unroll
            for (int k = 0; k < 9; ++k) j[k] *= albedo;
            // intensity(color) / 255.0f in float (src/color_util.cpp:41-46, lighting_svsh.cpp:230)
            const uchar4 c = g.rgb[v];
            const float lumf = FD(FA(FA(FM(0.299f, static_cast<float>(c.x)), FM(0.587f, static_cast<float>(c.y))), FM(0.114f, static_cast<float>(c.z))), 255.0f);
            const double lum = static_cast<double>(lumf);
            double w = 1.0;
            if (weighted)
            {
                // SDFOperators::sdfToWeight (src/sdf/operators.cpp:142-147)
                const double T = static_cast<double>(g.truncation);
                w = fmin(fmax(1.0 - fmin(fabs(sdf), T) / T, 0.01), 1.0);
            }
            int q = 0;
#pragma unroll
            for (int a = 0; a < 9; ++a)
#pragma unroll
                for (int b = a; b < 9; ++b) vals[q++] = w * j[a] * j[b];
#pragma unroll
            for (int a = 0; a < 9; ++a) vals[45 + a] = w * lum * j[a];
            vals[54] = w * lum * lum;
            vals[55] = w;
            vals[56] = 1.0;
        }
    }
    // one reduction per distinct subvolume of the warp (voxels are brick-ordered: almost always one)
    unsigned todo = __ballot_sync(0xffffffffu, sid >= 0);
    while (todo)
    {
        const int leader = __ffs(todo) - 1;
        const int cur = __shfl_sync(0xffffffffu, sid, leader);
        const bool mine = sid == cur;
        todo &= ~__ballot_sync(0xffffffffu, mine);
        double keep0 = 0.0, keep1 = 0.0;
#pragma unroll
        for (int q = 0; q < kLightAcc; ++q)
        {
            const double t = warp_allsum(mine ? vals[q] : 0.0);
            if (lane == (q & 31)) { if (q < 32) keep0 = t; else keep1 = t; }
        }
        double* dst = acc + static_cast<int64_t>(cur) * kLightAcc;
        atomicAdd(dst + lane, keep0);
        if (32 + lane < kLightAcc) atomicAdd(dst + 32 + lane, keep1);
    }
}

// ----------------------------------------------------------------------------------------------
// single-CTA ceres::Solve on the reduced system
// ----------------------------------------------------------------------------------------------
struct LightSolveWork
{
    int S;
    const double* acc;          // [S][kLightAcc]
    const int32_t* nbr;         // [6][S]
    double* H;                  // [S][81] normalised data-term blocks
    double* Minv;               // [S][81] inverted preconditioner blocks
    double* g;                  // [M]  J^T l  (unscaled)
    double* scale;              // [M]  Jacobi column scaling
    double* diag;               // [M]  clamped squared column norms of the scaled Jacobian
    double* D2;                 // [M]  diag / radius
    double* gU;                 // [M]  unscaled gradient A x - g at the current point
    double* x; double* b; double* xs; double* r; double* z; double* p; double* q; double* t; double* w;   // [M] each
    int* deg;                   // [S]
    I3DLightingInfo* info;
};

__device__ __forceinline__ double block_allsum(double v, double* smem /* [33] */)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    v = warp_allsum(v);
    __syncthreads();
    if (lane == 0) smem[wid] = v;
    __syncthreads();
    double s = 0.0;
    const int nw = blockDim.x >> 5;
    for (int i = 0; i < nw; ++i) s += smem[i];      // same order in every thread: identical value everywhere
    return s;
}
__device__ __forceinline__ double block_allmax(double v, double* smem)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if (lane == 0) smem[wid] = v;
    __syncthreads();
    double s = smem[0];
    const int nw = blockDim.x >> 5;
    for (int i = 1; i < nw; ++i) s = fmax(s, smem[i]);
    return s;
}

// out = A in with A = blockdiag(H) + 2 wr (Deg - Adj) (x) I9; `in` must be visible to the block (sync before)
__device__ __forceinline__ double light_apply_row(const LightSolveWork& W, double wr2, const double* in, int j)
{
    const int s = j / 9, k = j - 9 * s;
    const double* Hs = W.H + static_cast<int64_t>(s) * 81 + 9 * k;
    const double* v = in + 9 * s;
    double a = 0.0;
#pragma unroll
    for (int c = 0; c < 9; ++c) a += Hs[c] * v[c];
    double nb = 0.0;
#pragma unroll
    for (int d = 0; d < 6; ++d) { const int o = W.nbr[static_cast<int64_t>(d) * W.S + s]; if (o >= 0) nb += in[9 * o + k]; }
    return a + wr2 * (static_cast<double>(W.deg[s]) * in[j] - nb);
}

// 9x9 SPD inverse by Cholesky (BlockJacobiPreconditioner: llt().solve(Identity)); false if not positive definite
__device__ inline bool spd_inverse9(const double* A, double* inv)
{
    double L[81];
    for (int i = 0; i < 9; ++i)
        for (int j = 0; j <= i; ++j)
        {
            double s = A[i * 9 + j];
            for (int k = 0; k < j; ++k) s -= L[i * 9 + k] * L[j * 9 + k];
            if (i == j) { if (!(s > 0.0)) return false; L[i * 9 + i] = sqrt(s); }
            else L[i * 9 + j] = s / L[j * 9 + j];
        }
    for (int c = 0; c < 9; ++c)
    {
        double y[9], xv[9];
        for (int i = 0; i < 9; ++i)
        {
            double s = (i == c) ? 1.0 : 0.0;
            for (int k = 0; k < i; ++k) s -= L[i * 9 + k] * y[k];
            y[i] = s / L[i * 9 + i];
        }
        for (int i = 8; i >= 0; --i)
        {
            double s = y[i];
            for (int k = i + 1; k < 9; ++k) s -= L[k * 9 + i] * xv[k];
            xv[i] = s / L[i * 9 + i];
        }
        for (int i = 0; i < 9; ++i) inv[i * 9 + c] = xv[i];
    }
    return true;
}

__global__ void __launch_bounds__(kLightSolveThreads) k_svsh_solve(LightSolveWork W, I3DLightingParams P)
{
    __shared__ double red[33];
    __shared__ int s_fail;
    const int tid = threadIdx.x, T = blockDim.x;
    const int S = W.S, M = 9 * S;
    if (tid == 0) s_fail = 0;

    // ---- problem assembly: loss weights (lighting_svsh.cpp:298-318), blocks, degrees ----
    double sw = 0.0, sc = 0.0, srows = 0.0, sdeg = 0.0;
    for (int s = tid; s < S; s += T)
    {
        const double* a = W.acc + static_cast<int64_t>(s) * kLightAcc;
        sw += a[55]; sc += a[54]; srows += a[56];
        int d = 0;
        for (int k = 0; k < 6; ++k) d += W.nbr[static_cast<int64_t>(k) * S + s] >= 0;
        W.deg[s] = d; sdeg += d;
    }
    const double sum_w = block_allsum(sw, red);
    const double n_rows = block_allsum(srows, red);
    const double n_pairs = block_allsum(sdeg, red);
    const double data_loss = sum_w > 0.0 ? 1.0 / sum_w : 1.0;
    const double c0 = data_loss * block_allsum(sc, red);
    const double wr = n_pairs > 0.0 ? P.lambda_reg / n_pairs : 0.0;
    const double wr2 = 2.0 * wr;            // every undirected pair is added in both directions
    for (int s = tid; s < S; s += T)
    {
        const double* a = W.acc + static_cast<int64_t>(s) * kLightAcc;
        double* Hs = W.H + static_cast<int64_t>(s) * 81;
        int q = 0;
        for (int i = 0; i < 9; ++i)
            for (int j = i; j < 9; ++j) { const double h = data_loss * a[q++]; Hs[9 * i + j] = h; Hs[9 * j + i] = h; }
        for (int i = 0; i < 9; ++i) W.g[9 * s + i] = data_loss * a[45 + i];
    }
    __syncthreads();
    // ---- iteration 0: x = 0, cost, Jacobi scaling, gradient ----
    double gmax_l = 0.0;
    for (int j = tid; j < M; j += T)
    {
        const int s = j / 9, k = j - 9 * s;
        const double colsq = W.H[static_cast<int64_t>(s) * 81 + 10 * k] + wr2 * static_cast<double>(W.deg[s]);
        const double sc_j = 1.0 / (1.0 + sqrt(colsq));
        W.scale[j] = sc_j;
        W.diag[j] = fmin(fmax(colsq * sc_j * sc_j, P.min_lm_diagonal), P.max_lm_diagonal);
        W.x[j] = 0.0;
        W.gU[j] = -W.g[j];
        gmax_l = fmax(gmax_l, fabs(W.g[j]));
    }
    double gmax = block_allmax(gmax_l, red);
    double cost = 0.5 * c0;
    const double cost_initial = cost;
    double x_norm = 0.0;
    double radius = P.initial_trust_region_radius, decrease_factor = 2.0;
    int invalid_steps = 0, termination = 1, it = 0, successful = 0, cg_total = 0;

    for (;;)
    {
        // FinalizeIterationAndCheckIfMinimizerCanContinue
        if (it >= P.max_iterations) { termination = 1; break; }
        if (gmax <= P.gradient_tolerance) { termination = 0; break; }
        if (radius <= P.min_trust_region_radius) { termination = 0; break; }
        ++it;
        // LevenbergMarquardtStrategy::ComputeStep: D = sqrt(diag / radius); right-hand side b = J~^T f
        for (int j = tid; j < M; j += T)
        {
            W.D2[j] = W.diag[j] / radius;
            const double bj = W.scale[j] * W.gU[j];
            W.b[j] = bj; W.r[j] = bj; W.xs[j] = 0.0;
        }
        __syncthreads();
        // BlockJacobiPreconditioner::Update
        for (int s = tid; s < S; s += T)
        {
            double B[81];
            const double* Hs = W.H + static_cast<int64_t>(s) * 81;
            for (int i = 0; i < 9; ++i)
                for (int j = 0; j < 9; ++j)
                {
                    double h = Hs[9 * i + j];
                    if (i == j) h += wr2 * static_cast<double>(W.deg[s]);
                    h *= W.scale[9 * s + i] * W.scale[9 * s + j];
                    if (i == j) h += W.D2[9 * s + i];
                    B[9 * i + j] = h;
                }
            if (!spd_inverse9(B, W.Minv + static_cast<int64_t>(s) * 81)) s_fail = 1;
        }
        __syncthreads();
        if (s_fail) { termination = 2; break; }
        // ---- ConjugateGradientsSolver on (J~^T J~ + D^2) y = b, y0 = 0 ----
        double bb = 0.0;
        for (int j = tid; j < M; j += T) bb += W.b[j] * W.b[j];
        const double norm_b = sqrt(block_allsum(bb, red));
        int cg_it = 0; bool cg_failed = false;
        if (norm_b != 0.0)
        {
            double rho = 1.0, Q0 = 0.0;
            for (cg_it = 1;; ++cg_it)
            {
                double part = 0.0;
                for (int j = tid; j < M; j += T)
                {
                    const int s = j / 9, k = j - 9 * s;
                    const double* Mi = W.Minv + static_cast<int64_t>(s) * 81 + 9 * k;
                    const double* rv = W.r + 9 * s;
                    double zz = 0.0;
#pragma unroll
                    for (int c = 0; c < 9; ++c) zz += Mi[c] * rv[c];
                    W.z[j] = zz;
                    part += W.r[j] * zz;
                }
                const double last_rho = rho;
                rho = block_allsum(part, red);
                if (rho == 0.0 || isinf(rho)) { cg_failed = true; break; }
                double beta = 0.0;
                if (cg_it > 1)
                {
                    beta = rho / last_rho;
                    if (beta == 0.0 || isinf(beta)) { cg_failed = true; break; }
                }
                for (int j = tid; j < M; j += T)
                {
                    const double pj = cg_it == 1 ? W.z[j] : W.z[j] + beta * W.p[j];
                    W.p[j] = pj;
                    W.t[j] = W.scale[j] * pj;
                }
                __syncthreads();
                part = 0.0;
                for (int j = tid; j < M; j += T)
                {
                    const double qj = W.scale[j] * light_apply_row(W, wr2, W.t, j) + W.D2[j] * W.p[j];
                    W.q[j] = qj;
                    part += W.p[j] * qj;
                }
                const double pq = block_allsum(part, red);
                if (pq <= 0.0 || isinf(pq)) break;            // NO_CONVERGENCE: the step is still used
                const double alpha = rho / pq;
                if (isinf(alpha)) { cg_failed = true; break; }
                const bool refresh = (cg_it % P.residual_reset_period) == 0;
                for (int j = tid; j < M; j += T)
                {
                    const double xj = W.xs[j] + alpha * W.p[j];
                    W.xs[j] = xj;
                    if (refresh) W.t[j] = W.scale[j] * xj; else W.r[j] -= alpha * W.q[j];
                }
                if (refresh)
                {
                    __syncthreads();
                    for (int j = tid; j < M; j += T) W.r[j] = W.b[j] - (W.scale[j] * light_apply_row(W, wr2, W.t, j) + W.D2[j] * W.xs[j]);
                }
                part = 0.0;
                for (int j = tid; j < M; j += T) part -= W.xs[j] * (W.b[j] + W.r[j]);
                const double Q1 = block_allsum(part, red);
                const double zeta = cg_it * (Q1 - Q0) / Q1;
                if (zeta < P.eta && cg_it >= P.min_linear_solver_iterations) break;
                Q0 = Q1;
                if (cg_it >= P.max_linear_solver_iterations) break;
            }
        }
        cg_total += cg_it;
        // step = -solution; model_cost_change = -(J~ s).(f + J~ s / 2) = -(s.b + s.(A~ s) / 2)
        double bad = 0.0;
        for (int j = tid; j < M; j += T)
        {
            const double sj = -W.xs[j];
            W.xs[j] = sj;
            W.t[j] = W.scale[j] * sj;         // = delta (unscaled step)
            if (!isfinite(sj)) bad = 1.0;
        }
        const bool finite_step = block_allsum(bad, red) == 0.0;     // also orders the writes of t
        bool step_valid = !cg_failed && finite_step;
        double model_cost_change = 0.0;
        if (step_valid)
        {
            double part = 0.0;
            for (int j = tid; j < M; j += T)
            {
                const double Ad = light_apply_row(W, wr2, W.t, j);     // A delta
                W.w[j] = Ad;
                part += W.xs[j] * W.b[j] + 0.5 * W.t[j] * Ad;          // s.b + (delta . A delta) / 2
            }
            model_cost_change = -block_allsum(part, red);
            step_valid = model_cost_change > 0.0;
        }
        if (!step_valid)
        {
            if (++invalid_steps >= P.max_consecutive_invalid_steps) { termination = 2; break; }
            radius *= 0.5;
            continue;
        }
        invalid_steps = 0;
        // candidate: x + delta; gradient there gU + A delta; cost = (x.(gU - g) + c) / 2
        double p_step = 0.0, p_cost = 0.0;
        for (int j = tid; j < M; j += T)
        {
            const double cx = W.x[j] + W.t[j];
            const double dj = W.x[j] - cx;
            p_step += dj * dj;
            p_cost += cx * (W.gU[j] + W.w[j] - W.g[j]);
        }
        const double step_norm = sqrt(block_allsum(p_step, red));
        const double cand = 0.5 * (block_allsum(p_cost, red) + c0);
        if (step_norm <= P.parameter_tolerance * (x_norm + P.parameter_tolerance)) { termination = 0; break; }
        const double cost_change = cost - cand;
        if (fabs(cost_change) <= P.function_tolerance * cost) { termination = 0; break; }
        const double rho_q = cost_change / model_cost_change;
        if (rho_q > P.min_relative_decrease)
        {
            double p_x = 0.0, p_g = 0.0;
            for (int j = tid; j < M; j += T)
            {
                const double cx = W.x[j] + W.t[j];
                const double gj = W.gU[j] + W.w[j];
                W.x[j] = cx; W.gU[j] = gj;
                p_x += cx * cx;
                p_g = fmax(p_g, fabs(gj));
            }
            x_norm = sqrt(block_allsum(p_x, red));
            gmax = block_allmax(p_g, red);
            cost = cand;
            const double u = 2.0 * rho_q - 1.0;
            radius = radius / fmax(1.0 / 3.0, 1.0 - u * u * u);
            radius = fmin(P.max_trust_region_radius, radius);
            decrease_factor = 2.0;
            ++successful;
        }
        else { radius = radius / decrease_factor; decrease_factor *= 2.0; }
    }
    __syncthreads();
    if (tid == 0)
    {
        I3DLightingInfo& I = *W.info;
        I.num_subvolumes = S;
        I.num_data_rows = static_cast<int64_t>(n_rows + 0.5);
        I.num_reg_pairs = static_cast<int64_t>(n_pairs + 0.5);
        I.sum_data_weights = sum_w;
        I.cost_initial = cost_initial; I.cost_final = cost;
        I.trust_region_radius = radius;
        I.lm_iterations = it; I.num_successful_steps = successful; I.cg_iterations_total = cg_total;
        I.termination = termination; I.usable = termination != 2;
    }
}

// computeVoxelShCoeffs -> Subvolumes::interpolate(linear).  sh_soa is the engine's [9][n] layout.
__global__ void __launch_bounds__(kThreads) k_svsh_interpolate(GridView g, SubvolGrid sg, double thres_shell, const double* __restrict__ sub_sh /* [S][9] */,
                                                                 double* __restrict__ sh_soa, uint8_t* __restrict__ has)
{
    const int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (v >= g.n) return;
    double avg[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) avg[k] = 0.0;
    const bool use = g.weight[v] > 0.0f && !(fabs(g.sdf[v]) > thres_shell);
    if (use) svsh_blend(g, v, sg, sub_sh, avg);
#pragma unroll
    for (int k = 0; k < 9; ++k) sh_soa[static_cast<int64_t>(k) * g.n + v] = avg[k];
    has[v] = use ? 1 : 0;
}

__global__ void k_untranspose_sh(int64_t n, const double* __restrict__ sh_soa, double* __restrict__ sh_aos)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= 9 * n) return;
    const int64_t v = i / 9; const int k = static_cast<int>(i - 9 * v);
    sh_aos[i] = sh_soa[static_cast<int64_t>(k) * n + v];
}

} // namespace i3d
