/*
 * i3d_math.cuh — scalar math of the E_g (gradient-of-shading) residual and its hand-derived
 * Jacobian row, shared by the Jacobian-build and cost kernels.
 *
 * What is computed follows the reference functor (libintrinsic3d/include/nv/refinement/
 * shading_cost.h:85-198 and its helpers: include/nv/sdf/operators.h:49-86,
 * include/nv/refinement/cost.h:80-127, include/nv/camera.h:96-116, include/nv/shading.h:53-148)
 * and the Ceres pieces it calls (AngleAxisRotatePoint, BiCubicInterpolator over a clamped
 * Grid2D<float>).  HOW it is computed is not: the reference differentiates the functor with
 * forward-mode Jets (8 passes of 4 lanes per row); here the 29-column row is assembled from a
 * closed-form chain rule (SURVEY.md Appendix A) in ONE pass per sample point:
 *     dr/dtheta = sum_i e_i (dS_i/dtheta - dL_i/dtheta),  e_j = d_j / r, e_0 = -sum_j e_j.
 *
 * Everything is templated on the scalar type: the primal (validity + residual value) is
 * evaluated in double, the derivative pass in float (I3D_DERIV_T).
 *
 * The header is also compilable by a host compiler (tests/native/) with I3D_HD empty, which is
 * how the analytic row is checked against the oracle's Jets without a GPU.
 */
#pragma once

#ifndef I3D_HD
#ifdef __CUDACC__
#define I3D_HD __host__ __device__ __forceinline__
#else
#define I3D_HD inline
#endif
#endif

#include <math.h>

namespace i3d
{

// stencil: sdf parameter p -> neighbour slot. Parameter order of the reference (shading_cost.h:89-98):
// 0:(0,0,0) 1:(0,1,0) 2:(0,2,0) 3:(0,1,1) 4:(0,0,1) 5:(0,0,2) 6:(1,0,0) 7:(1,1,0) 8:(1,0,1) 9:(2,0,0)
// point i uses quadruple (s, s+x, s+y, s+z): kQuad[i][.] indexes the 10 sdf parameters.
// point 0 = v, 1 = v+x, 2 = v+y, 3 = v+z
#define I3D_QUAD(i, j) (((i) == 0) ? (((j) == 0) ? 0 : ((j) == 1) ? 6 : ((j) == 2) ? 1 : 4) \
                      : ((i) == 1) ? (((j) == 0) ? 6 : ((j) == 1) ? 9 : ((j) == 2) ? 7 : 8) \
                      : ((i) == 2) ? (((j) == 0) ? 1 : ((j) == 1) ? 7 : ((j) == 2) ? 2 : 3) \
                                   : (((j) == 0) ? 4 : ((j) == 1) ? 8 : ((j) == 2) ? 3 : 5))

template <class T> struct Num;
template <> struct Num<double>
{
    static I3D_HD double sqrt_(double x) { return sqrt(x); }
    static I3D_HD double floor_(double x) { return floor(x); }
    static I3D_HD void sincos_(double x, double* s, double* c) { *s = sin(x); *c = cos(x); }
#ifdef __CUDA_ARCH__
    static I3D_HD double rsqrt_(double x) { return rsqrt(x); }
#else
    static I3D_HD double rsqrt_(double x) { return 1.0 / sqrt(x); }
#endif
};
template <> struct Num<float>
{
    static I3D_HD float sqrt_(float x) { return sqrtf(x); }
    static I3D_HD float floor_(float x) { return floorf(x); }
    static I3D_HD void sincos_(float x, float* s, float* c) { *s = sinf(x); *c = cosf(x); }
#ifdef __CUDA_ARCH__
    static I3D_HD float rsqrt_(float x) { return rsqrtf(x); }
#else
    static I3D_HD float rsqrt_(float x) { return 1.0f / sqrtf(x); }
#endif
};

// camera-side constants shared by every row of one frame / one launch
template <class T>
struct CamParams
{
    T fx, fy, cx, cy;      // intrinsics already multiplied by pyr_scale
    T k1, k2, k3, p1, p2;  // distortion
    T pyr_scale;
    int w, h;
};

// Catmull-Rom cubic convolution (ceres::CubicHermiteSpline): value and derivative
template <class T>
I3D_HD void cubic(T p0, T p1, T p2, T p3, T x, T* f, T* dfdx)
{
    const T a = T(0.5) * (-p0 + T(3.0) * p1 - T(3.0) * p2 + p3);
    const T b = T(0.5) * (T(2.0) * p0 - T(5.0) * p1 + T(4.0) * p2 - p3);
    const T c = T(0.5) * (-p0 + p2);
    *f = p1 + x * (c + x * (b + x * a));
    *dfdx = c + x * (T(2.0) * b + T(3.0) * a * x);
}

// ceres::BiCubicInterpolator::Evaluate(r = v, c = u) on Grid2D<float,1,true,true> (indices clamped).
// Returns f, df/du (column direction), df/dv (row direction).
template <class T>
I3D_HD void bicubic(const float* __restrict__ img, int w, int h, T u, T v, T* f, T* dfdu, T* dfdv)
{
    const T fu = Num<T>::floor_(u), fv = Num<T>::floor_(v);
    const int col = static_cast<int>(fu), row = static_cast<int>(fv);
    const T xu = u - fu, xv = v - fv;
    int cc[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { int c = col - 1 + j; c = c < 0 ? 0 : c; cc[j] = c > w - 1 ? w - 1 : c; }
    T fr[4], dfc[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
    {
        int rr = row - 1 + i; rr = rr < 0 ? 0 : rr; rr = rr > h - 1 ? h - 1 : rr;
        const float* line = img + static_cast<size_t>(rr) * w;
#ifdef __CUDA_ARCH__
        const T p0 = T(__ldg(line + cc[0])), p1 = T(__ldg(line + cc[1])), p2 = T(__ldg(line + cc[2])), p3 = T(__ldg(line + cc[3]));
#else
        const T p0 = T(line[cc[0]]), p1 = T(line[cc[1]]), p2 = T(line[cc[2]]), p3 = T(line[cc[3]]);
#endif
        cubic<T>(p0, p1, p2, p3, xu, &fr[i], &dfc[i]);
    }
    cubic<T>(fr[0], fr[1], fr[2], fr[3], xv, f, dfdv);
    T unused;
    cubic<T>(dfc[0], dfc[1], dfc[2], dfc[3], xv, dfdu, &unused);
}

// Pose context: everything of AngleAxisRotatePoint that does not depend on the point, computed
// once per row (the reference recomputes sin/cos for each of the 4 sample points).
template <class T>
struct PoseCtx
{
    T w[3];        // unit axis (general branch) or the raw angle-axis vector (small-angle branch)
    T st, ct, ti;  // sin(theta), cos(theta), 1/theta
    T t[3];
    T R[9];        // rotation matrix (row-major), used for dL/dX = dL/dY * R
    bool small;    // theta^2 <= DBL_EPSILON: ceres uses Y = X + omega x X
};

I3D_HD void pose_ctx_make(const double* __restrict__ pose, PoseCtx<double>* c)
{
    const double a0 = pose[0], a1 = pose[1], a2 = pose[2];
    const double theta2 = a0 * a0 + a1 * a1 + a2 * a2;
    c->t[0] = pose[3]; c->t[1] = pose[4]; c->t[2] = pose[5];
    if (theta2 > 2.220446049250313e-16)
    {
        const double theta = sqrt(theta2);
        c->small = false;
        c->st = sin(theta); c->ct = cos(theta); c->ti = 1.0 / theta;
        c->w[0] = a0 * c->ti; c->w[1] = a1 * c->ti; c->w[2] = a2 * c->ti;
        const double omc = 1.0 - c->ct;
        const double* w = c->w;
        c->R[0] = c->ct + omc * w[0] * w[0];          c->R[1] = -c->st * w[2] + omc * w[0] * w[1];  c->R[2] = c->st * w[1] + omc * w[0] * w[2];
        c->R[3] = c->st * w[2] + omc * w[1] * w[0];   c->R[4] = c->ct + omc * w[1] * w[1];          c->R[5] = -c->st * w[0] + omc * w[1] * w[2];
        c->R[6] = -c->st * w[1] + omc * w[2] * w[0];  c->R[7] = c->st * w[0] + omc * w[2] * w[1];   c->R[8] = c->ct + omc * w[2] * w[2];
    }
    else
    {
        c->small = true;
        c->st = 0.0; c->ct = 1.0; c->ti = 0.0;
        c->w[0] = a0; c->w[1] = a1; c->w[2] = a2;
        c->R[0] = 1.0; c->R[1] = -a2;  c->R[2] = a1;
        c->R[3] = a2;  c->R[4] = 1.0;  c->R[5] = -a0;
        c->R[6] = -a1; c->R[7] = a0;   c->R[8] = 1.0;
    }
}

template <class T>
I3D_HD void pose_ctx_cast(const PoseCtx<double>& s, PoseCtx<T>* d)
{
#pragma unroll
    for (int k = 0; k < 3; ++k) { d->w[k] = T(s.w[k]); d->t[k] = T(s.t[k]); }
#pragma unroll
    for (int k = 0; k < 9; ++k) d->R[k] = T(s.R[k]);
    d->st = T(s.st); d->ct = T(s.ct); d->ti = T(s.ti); d->small = s.small;
}

// ceres::AngleAxisRotatePoint + translation.  Also returns dY/domega (3x3, row-major:
// dY_r / domega_c) if D != nullptr.
template <class T>
I3D_HD void transform_point(const PoseCtx<T>& pc, const T X[3], T Y[3], T* D /* 9 or nullptr */)
{
    const T w0 = pc.w[0], w1 = pc.w[1], w2 = pc.w[2];
    const T c0 = w1 * X[2] - w2 * X[1], c1 = w2 * X[0] - w0 * X[2], c2 = w0 * X[1] - w1 * X[0];   // w x X
    if (!pc.small)
    {
        const T st = pc.st, ct = pc.ct, ti = pc.ti;
        const T wd = w0 * X[0] + w1 * X[1] + w2 * X[2];
        const T tmp = wd * (T(1.0) - ct);
        Y[0] = X[0] * ct + c0 * st + w0 * tmp;
        Y[1] = X[1] * ct + c1 * st + w1 * tmp;
        Y[2] = X[2] * ct + c2 * st + w2 * tmp;
        if (D)
        {
            // Y = c X + s (w x X) + (1-c)(w.X) w ;  theta-part a (x) w^T, w-part B (I - w w^T)/theta
            const T a[3] = {-st * X[0] + ct * c0 + st * wd * w0, -st * X[1] + ct * c1 + st * wd * w1, -st * X[2] + ct * c2 + st * wd * w2};
            const T omc = T(1.0) - ct;
            // B = s * (-[X]x) + (1-c) * (w X^T + (w.X) I)
            T B[9];
            B[0] = omc * (w0 * X[0] + wd);       B[1] = st * X[2] + omc * w0 * X[1];  B[2] = -st * X[1] + omc * w0 * X[2];
            B[3] = -st * X[2] + omc * w1 * X[0]; B[4] = omc * (w1 * X[1] + wd);       B[5] = st * X[0] + omc * w1 * X[2];
            B[6] = st * X[1] + omc * w2 * X[0];  B[7] = -st * X[0] + omc * w2 * X[1]; B[8] = omc * (w2 * X[2] + wd);
            const T w[3] = {w0, w1, w2};
#pragma unroll
            for (int r = 0; r < 3; ++r)
            {
                const T bw = B[3 * r] * w0 + B[3 * r + 1] * w1 + B[3 * r + 2] * w2;   // (B w)_r
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    D[3 * r + c] = a[r] * w[c] + (B[3 * r + c] - bw * w[c]) * ti;
            }
        }
    }
    else
    {
        Y[0] = X[0] + c0; Y[1] = X[1] + c1; Y[2] = X[2] + c2;
        if (D)
        {
            // Y = X + omega x X  =>  dY/domega = -[X]x
            D[0] = T(0);   D[1] = X[2];  D[2] = -X[1];
            D[3] = -X[2];  D[4] = T(0);  D[5] = X[0];
            D[6] = X[1];   D[7] = -X[0]; D[8] = T(0);
        }
    }
    Y[0] += pc.t[0]; Y[1] += pc.t[1]; Y[2] += pc.t[2];
}

// un-normalised SH basis in the reference's order (include/nv/shading.h:57-65): value and gradient wrt n
template <class T>
I3D_HD T sh_eval(const T* __restrict__ c, const T n[3], T grad[3])
{
    const T x = n[0], y = n[1], z = n[2];
    T s = c[0];
    s += c[1] * y;
    s += c[2] * z;
    s += c[3] * x;
    s += c[4] * (x * y);
    s += c[5] * (y * z);
    s += c[6] * ((-(x * x)) - (y * y) + T(2.0) * (z * z));
    s += c[7] * (x * z);
    s += c[8] * ((x * x) - (y * y));
    if (grad)
    {
        grad[0] = c[3] + c[4] * y - T(2.0) * c[6] * x + c[7] * z + T(2.0) * c[8] * x;
        grad[1] = c[1] + c[4] * x + c[5] * z - T(2.0) * c[6] * y - T(2.0) * c[8] * y;
        grad[2] = c[2] + c[5] * y + T(4.0) * c[6] * z + c[7] * x;
    }
    return s;
}

// Primal of one sample point: shading S, luminance L with its image-space gradient (Lu = dL/du,
// Lv = dL/dv, by-products of the bicubic), in-bounds flag.
// q = (s, s+x, s+y, s+z); coord = integer voxel coordinate of the point; pose = (omega, t).
template <class T>
I3D_HD bool point_primal(const T q[4], T albedo, const int coord[3], T voxel_size, const PoseCtx<T>& pose,
                         const CamParams<T>& cam, const float* __restrict__ img, const T* __restrict__ sh, T* S, T* L, T* Lu, T* Lv)
{
    T g[3] = {q[1] - q[0], q[2] - q[0], q[3] - q[0]};
    const T len2 = g[0] * g[0] + g[1] * g[1] + g[2] * g[2];
    if (len2 > T(0)) { const T il = Num<T>::rsqrt_(len2); g[0] *= il; g[1] *= il; g[2] *= il; }   // normalised iff length > 0
    T X[3], Y[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) X[k] = T(coord[k]) * voxel_size - g[k] * q[0];
    transform_point<T>(pose, X, Y, nullptr);
    const T iz = T(1.0) / Y[2];
    const T x = Y[0] * iz, y = Y[1] * iz;
    const T r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
    const T dc = T(1.0) + cam.k1 * r2 + cam.k2 * r4 + cam.k3 * r6;
    const T xd = x * dc + T(2.0) * cam.p1 * x * y + cam.p2 * (r2 + T(2.0) * x * x);
    const T yd = y * dc + T(2.0) * cam.p2 * xd * y + cam.p1 * (r2 + T(2.0) * y * y);
    const T u = cam.fx * xd + cam.cx, v = cam.fy * yd + cam.cy;
    // same comparison as CameraT::project (NaN => comparisons false => "inside", caught by the finite test later)
    if (u < T(0) || u > T(cam.w - 1) || v < T(0) || v > T(cam.h - 1)) return false;
    bicubic<T>(img, cam.w, cam.h, u, v, L, Lu, Lv);
    *S = albedo * sh_eval<T>(sh, g, nullptr);
    return true;
}

// Derivative contribution of one sample point, accumulated with weight e into the 29-column row:
//   row[quad params] += e * (dS/dq - dL/dq);  row[10 + i] += e * sigma;
//   row[14..19] -= e * dL/dpose; row[20..23] -= e * dL/dintr; row[24..28] -= e * dL/ddist
// `point` selects which sdf/albedo columns the quadruple maps to.
template <class T, int POINT>
I3D_HD void point_deriv(const T q[4], T albedo, const int coord[3], T voxel_size, const PoseCtx<T>& pose,
                        const CamParams<T>& cam, const T* __restrict__ sh, T Lu, T Lvv, T e, T* __restrict__ row)
{
    const T s = q[0];
    T g[3] = {q[1] - s, q[2] - s, q[3] - s};
    const T len2 = g[0] * g[0] + g[1] * g[1] + g[2] * g[2];
    // dn/d(sx,sy,sz) = P (3x3), dn/ds = -P*1
    T P[9];
    if (len2 > T(0))
    {
        const T il = Num<T>::rsqrt_(len2);
        g[0] *= il; g[1] *= il; g[2] *= il;
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) P[3 * r + c] = ((r == c ? T(1.0) : T(0.0)) - g[r] * g[c]) * il;
    }
    else
    {
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) P[3 * r + c] = (r == c ? T(1.0) : T(0.0));
    }
    T gs[3];
    const T sigma = sh_eval<T>(sh, g, gs);
    T X[3], Y[3], Dw[9];
#pragma unroll
    for (int k = 0; k < 3; ++k) X[k] = T(coord[k]) * voxel_size - g[k] * s;
    transform_point<T>(pose, X, Y, Dw);
    const T iz = T(1.0) / Y[2];
    const T x = Y[0] * iz, y = Y[1] * iz;
    const T r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
    const T dc = T(1.0) + cam.k1 * r2 + cam.k2 * r4 + cam.k3 * r6;
    const T dcp = cam.k1 + T(2.0) * cam.k2 * r2 + T(3.0) * cam.k3 * r4;      // d(dc)/d(r2)
    const T xd = x * dc + T(2.0) * cam.p1 * x * y + cam.p2 * (r2 + T(2.0) * x * x);
    const T yd = y * dc + T(2.0) * cam.p2 * xd * y + cam.p1 * (r2 + T(2.0) * y * y);
    // (Lu, Lvv) = image gradient (dL/du, dL/dv) at the projected point, taken from the double-precision
    // primal pass: the derivative pass never samples the image.
    // d(xd,yd)/d(x,y)
    const T xdx = dc + T(2.0) * x * x * dcp + T(2.0) * cam.p1 * y + T(6.0) * cam.p2 * x;
    const T xdy = T(2.0) * x * y * dcp + T(2.0) * cam.p1 * x + T(2.0) * cam.p2 * y;
    const T ydx = T(2.0) * x * y * dcp + T(2.0) * cam.p2 * y * xdx + T(2.0) * cam.p1 * x;
    const T ydy = dc + T(2.0) * y * y * dcp + T(2.0) * cam.p2 * (y * xdy + xd) + T(6.0) * cam.p1 * y;
    // dL/d(x,y)
    const T gu = Lu * cam.fx, gv = Lvv * cam.fy;
    const T Lx = gu * xdx + gv * ydx;
    const T Ly = gu * xdy + gv * ydy;
    // dL/dY
    const T LY[3] = {Lx * iz, Ly * iz, -(Lx * x + Ly * y) * iz};
    // pose columns: rotation (dL/dY * dY/domega), translation (dL/dY)
#pragma unroll
    for (int c = 0; c < 3; ++c)
        row[14 + c] -= e * (LY[0] * Dw[c] + LY[1] * Dw[3 + c] + LY[2] * Dw[6 + c]);
#pragma unroll
    for (int c = 0; c < 3; ++c) row[17 + c] -= e * LY[c];
    // intrinsics (parameters live at full resolution: u = pyr_scale*(fx*xd + cx))
    row[20] -= e * (Lu * cam.pyr_scale * xd);
    row[21] -= e * (Lvv * cam.pyr_scale * yd);
    row[22] -= e * (Lu * cam.pyr_scale);
    row[23] -= e * (Lvv * cam.pyr_scale);
    // distortion k1,k2,k3,p1,p2
    {
        const T c2y = T(2.0) * cam.p2 * y;
        const T xk1 = x * r2, xk2 = x * r4, xk3 = x * r6, xp1 = T(2.0) * x * y, xp2 = r2 + T(2.0) * x * x;
        row[24] -= e * (gu * xk1 + gv * (y * r2 + c2y * xk1));
        row[25] -= e * (gu * xk2 + gv * (y * r4 + c2y * xk2));
        row[26] -= e * (gu * xk3 + gv * (y * r6 + c2y * xk3));
        row[27] -= e * (gu * xp1 + gv * ((r2 + T(2.0) * y * y) + c2y * xp1));
        row[28] -= e * (gu * xp2 + gv * (T(2.0) * xd * y + c2y * xp2));
    }
    // dL/dX = dL/dY * R
    const T LX[3] = {LY[0] * pose.R[0] + LY[1] * pose.R[3] + LY[2] * pose.R[6],
                     LY[0] * pose.R[1] + LY[1] * pose.R[4] + LY[2] * pose.R[7],
                     LY[0] * pose.R[2] + LY[1] * pose.R[5] + LY[2] * pose.R[8]};
    // dS/dn and dL/dn combined: X = h c - n s  =>  dX/dn = -s I ; plus explicit dX/ds = -n
    // v_n = albedo * grad_sigma - (-s) * LX  => contribution through n: (a*gs + s*LX) . dn/dq
    const T vn[3] = {albedo * gs[0] + s * LX[0], albedo * gs[1] + s * LX[1], albedo * gs[2] + s * LX[2]};
    // through dn/d(sx,sy,sz) = P columns
    const T d1 = vn[0] * P[0] + vn[1] * P[3] + vn[2] * P[6];
    const T d2 = vn[0] * P[1] + vn[1] * P[4] + vn[2] * P[7];
    const T d3 = vn[0] * P[2] + vn[1] * P[5] + vn[2] * P[8];
    // dn/ds = -(P col sums)  => -(d1+d2+d3); explicit dX/ds = -n => -dL: -( -n . LX ) = + n.LX
    const T d0 = -(d1 + d2 + d3) + (g[0] * LX[0] + g[1] * LX[1] + g[2] * LX[2]);
    row[I3D_QUAD(POINT, 0)] += e * d0;
    row[I3D_QUAD(POINT, 1)] += e * d1;
    row[I3D_QUAD(POINT, 2)] += e * d2;
    row[I3D_QUAD(POINT, 3)] += e * d3;
    row[10 + POINT] += e * sigma;
}

template <class T>
I3D_HD bool finite_(T x) { return (x - x) == T(0); }

// One E_g row: residual value in double (0.0 = NV_INVALID_RESIDUAL), and — if `row` is given and
// the residual is valid and non-zero — the raw 29-column Jacobian row d r / d theta in TD.
// sdf[10], alb[4] in the reference's parameter order; coord = voxel coordinate of the row's voxel.
template <class TD>
I3D_HD double eg_row(const double sdf[10], const double alb[4], const int coord[3], double voxel_size,
                     const PoseCtx<double>& pc, const CamParams<double>& cam, const float* __restrict__ img,
                     const double sh[9], TD* __restrict__ row)
{
    double S[4], L[4];
    float Lu[4], Lv[4];
    bool inb = true;
#pragma unroll
    for (int i = 0; i < 4; ++i)
    {
        const double q[4] = {sdf[I3D_QUAD(i, 0)], sdf[I3D_QUAD(i, 1)], sdf[I3D_QUAD(i, 2)], sdf[I3D_QUAD(i, 3)]};
        const int c[3] = {coord[0] + (i == 1), coord[1] + (i == 2), coord[2] + (i == 3)};
        S[i] = 0.0; L[i] = 0.0;
        double lu = 0.0, lv = 0.0;
        inb = point_primal<double>(q, alb[i], c, voxel_size, pc, cam, img, sh, &S[i], &L[i], &lu, &lv) && inb;
        Lu[i] = static_cast<float>(lu); Lv[i] = static_cast<float>(lv);
    }
    if (!inb) return 0.0;
    const double d1 = (S[1] - S[0]) - (L[1] - L[0]);
    const double d2 = (S[2] - S[0]) - (L[2] - L[0]);
    const double d3 = (S[3] - S[0]) - (L[3] - L[0]);
    const double r = sqrt(d1 * d1 + d2 * d2 + d3 * d3);
    if (!finite_(r)) return 0.0;
    if (row != nullptr && r != 0.0)
    {
        const double ir = 1.0 / r;
        const TD e[4] = {TD(-(d1 + d2 + d3) * ir), TD(d1 * ir), TD(d2 * ir), TD(d3 * ir)};
        PoseCtx<TD> pcd;
        pose_ctx_cast<TD>(pc, &pcd);
        CamParams<TD> cd;
        cd.fx = TD(cam.fx); cd.fy = TD(cam.fy); cd.cx = TD(cam.cx); cd.cy = TD(cam.cy);
        cd.k1 = TD(cam.k1); cd.k2 = TD(cam.k2); cd.k3 = TD(cam.k3); cd.p1 = TD(cam.p1); cd.p2 = TD(cam.p2);
        cd.pyr_scale = TD(cam.pyr_scale); cd.w = cam.w; cd.h = cam.h;
        TD shd[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) shd[k] = TD(sh[k]);
#pragma unroll
        for (int k = 0; k < 29; ++k) row[k] = TD(0);
        const TD vs = TD(voxel_size);
        {
            const TD q[4] = {TD(sdf[I3D_QUAD(0, 0)]), TD(sdf[I3D_QUAD(0, 1)]), TD(sdf[I3D_QUAD(0, 2)]), TD(sdf[I3D_QUAD(0, 3)])};
            const int c[3] = {coord[0], coord[1], coord[2]};
            point_deriv<TD, 0>(q, TD(alb[0]), c, vs, pcd, cd, shd, TD(Lu[0]), TD(Lv[0]), e[0], row);
        }
        {
            const TD q[4] = {TD(sdf[I3D_QUAD(1, 0)]), TD(sdf[I3D_QUAD(1, 1)]), TD(sdf[I3D_QUAD(1, 2)]), TD(sdf[I3D_QUAD(1, 3)])};
            const int c[3] = {coord[0] + 1, coord[1], coord[2]};
            point_deriv<TD, 1>(q, TD(alb[1]), c, vs, pcd, cd, shd, TD(Lu[1]), TD(Lv[1]), e[1], row);
        }
        {
            const TD q[4] = {TD(sdf[I3D_QUAD(2, 0)]), TD(sdf[I3D_QUAD(2, 1)]), TD(sdf[I3D_QUAD(2, 2)]), TD(sdf[I3D_QUAD(2, 3)])};
            const int c[3] = {coord[0], coord[1] + 1, coord[2]};
            point_deriv<TD, 2>(q, TD(alb[2]), c, vs, pcd, cd, shd, TD(Lu[2]), TD(Lv[2]), e[2], row);
        }
        {
            const TD q[4] = {TD(sdf[I3D_QUAD(3, 0)]), TD(sdf[I3D_QUAD(3, 1)]), TD(sdf[I3D_QUAD(3, 2)]), TD(sdf[I3D_QUAD(3, 3)])};
            const int c[3] = {coord[0], coord[1], coord[2] + 1};
            point_deriv<TD, 3>(q, TD(alb[3]), c, vs, pcd, cd, shd, TD(Lu[3]), TD(Lv[3]), e[3], row);
        }
    }
    return r;
}


// =====================================================================================================================
// Voxel-owned evaluation (round 2).  One thread owns ALL K rows of a voxel: everything of the functor that does not depend
// on the frame — the four normals, the four shading values S_i (hence the three differences S_j - S_0), the four iso-points
// X_i — is evaluated once per voxel (VoxelGeom, float64) instead of once per row, and the float side of the chain rule keeps
// (n_i, 1/l_i, a_i*grad sigma_i, sigma_i, s_i) in registers (VoxelDeriv).  Per frame only the rigid transform, the
// projection with distortion and the bicubic luminance lookup remain.
//
// Two algebraic changes against eg_row() above (same function, fewer instructions; both checked against the oracle's Jets
// in tests/test_eg_math.py):
//  * rotation columns:  dY/domega = -R [X]x Jr(omega)  (Jr = right Jacobian of SO(3), a per-FRAME constant), so
//        sum_i e_i dL_i/dY_i dY_i/domega = ( sum_i e_i X_i x (R^T dL_i/dY_i) )^T Jr
//    one cross product per point and ONE 3x3 product per row replace a 3x3 dY/domega per point.  In Ceres' small-angle
//    branch (Y = X + omega x X) the derivative is -[X]x exactly: Jr = I and dL/dY takes the place of R^T dL/dY.
//  * the bicubic is evaluated in weight form  L = sum_i wv_i sum_j wu_j p_ij  (Catmull-Rom weights; identical polynomial to
//    ceres::CubicHermiteSpline's Horner form); value and image gradient share the 16 converted taps.
// =====================================================================================================================

// per-frame constants of one pose (k_frame_pose): rotation in both precisions, Jr, the small-angle flag
struct FramePose
{
    double R[9];   // AngleAxisRotatePoint as a matrix (small-angle branch: I + [omega]x), row-major
    double t[3];
    float Rf[9];
    float Jr[9];   // right Jacobian of SO(3) (identity in the small-angle branch), row-major
    int small;
    int pad;
};
// k_eg_rows<ROWS_COST> stages F of these into shared memory; tests/test_gpu_lm_trial.py derives the staging boundary from this size
static_assert(sizeof(FramePose) == 176, "FramePose size changed: update the pose-table staging boundary and its test");

I3D_HD void frame_pose_make(const double* __restrict__ pose, FramePose* fp)
{
    PoseCtx<double> pc;
    pose_ctx_make(pose, &pc);
#pragma unroll
    for (int k = 0; k < 9; ++k) { fp->R[k] = pc.R[k]; fp->Rf[k] = static_cast<float>(pc.R[k]); }
#pragma unroll
    for (int k = 0; k < 3; ++k) fp->t[k] = pc.t[k];
    fp->small = pc.small ? 1 : 0; fp->pad = 0;
    double J[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
    if (!pc.small)
    {
        const double a0 = pose[0], a1 = pose[1], a2 = pose[2];
        const double th2 = a0 * a0 + a1 * a1 + a2 * a2, th = sqrt(th2);
        double ca, cb;   // (1 - cos th)/th^2, (th - sin th)/th^3
        if (th < 1e-2) { ca = 0.5 - th2 * (1.0 / 24.0) + th2 * th2 * (1.0 / 720.0); cb = (1.0 / 6.0) - th2 * (1.0 / 120.0) + th2 * th2 * (1.0 / 5040.0); }
        else { ca = (1.0 - pc.ct) / th2; cb = (th - pc.st) / (th2 * th); }
        // Jr = I - ca [w]x + cb [w]x^2 ;  [w]x^2 = w w^T - th^2 I
        J[0] = 1.0 + cb * (a0 * a0 - th2); J[1] = ca * a2 + cb * a0 * a1;      J[2] = -ca * a1 + cb * a0 * a2;
        J[3] = -ca * a2 + cb * a1 * a0;    J[4] = 1.0 + cb * (a1 * a1 - th2);  J[5] = ca * a0 + cb * a1 * a2;
        J[6] = ca * a1 + cb * a2 * a0;     J[7] = -ca * a0 + cb * a2 * a1;     J[8] = 1.0 + cb * (a2 * a2 - th2);
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) fp->Jr[k] = static_cast<float>(J[k]);
}

struct VoxelGeom      // frame-independent primal of the four sample points (float64)
{
    double X[4][3];   // iso-points in world coordinates
    double dS[3];     // S_j - S_0, j = 1..3
    I3D_HD double Xv(int i, int k) const { return X[i][k]; }
    I3D_HD double dSv(int j) const { return dS[j]; }
};
struct VoxelDeriv     // frame-independent float side of the chain rule
{
    float g[4][3];    // unit normals (raw zero vector if the gradient vanishes)
    float il[4];      // 1 / |gradient| (1 if it vanishes: dn/dq = I, as in point_deriv)
    float A[4][3];    // albedo_i * grad_n sigma(n_i)
    float sigma[4];   // sigma(n_i)
    float s[4];       // sdf value at point i
    float X0[3];      // voxel_size * coord of point 0
    float h;          // voxel size
    I3D_HD float gv(int i, int k) const { return g[i][k]; }
    I3D_HD float ilv(int i) const { return il[i]; }
    I3D_HD float Av(int i, int k) const { return A[i][k]; }
    I3D_HD float sigmav(int i) const { return sigma[i]; }
    I3D_HD float sv(int i) const { return s[i]; }
    I3D_HD float X0v(int k) const { return X0[k]; }
    I3D_HD float hv() const { return h; }
};

// The same state parked in shared memory, one column per thread ([field][thread]: lane-contiguous, conflict-free).  The kernels
// that keep ~70 registers of per-voxel state alive across the frame loop are occupancy-bound (168 registers, 11 warps per SM);
// read through these views (volatile: one LDS at each use, never hoisted back into registers for the whole loop) the state costs
// no registers between uses.
constexpr int kVoxelGeomWords = 15;      // doubles
constexpr int kVoxelDerivWords = 40;     // floats
struct VoxelGeomView
{
    const volatile double* p; int stride;     // p = column of this thread
    I3D_HD double Xv(int i, int k) const { return p[(3 * i + k) * stride]; }
    I3D_HD double dSv(int j) const { return p[(12 + j) * stride]; }
};
struct VoxelDerivView
{
    const volatile float* p; int stride;
    I3D_HD float gv(int i, int k) const { return p[(3 * i + k) * stride]; }
    I3D_HD float ilv(int i) const { return p[(12 + i) * stride]; }
    I3D_HD float Av(int i, int k) const { return p[(16 + 3 * i + k) * stride]; }
    I3D_HD float sigmav(int i) const { return p[(28 + i) * stride]; }
    I3D_HD float sv(int i) const { return p[(32 + i) * stride]; }
    I3D_HD float X0v(int k) const { return p[(36 + k) * stride]; }
    I3D_HD float hv() const { return p[39 * stride]; }
};
I3D_HD void voxel_geom_park(const VoxelGeom& vg, double* p, int stride)
{
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int k = 0; k < 3; ++k) p[(3 * i + k) * stride] = vg.X[i][k];
#pragma unroll
    for (int j = 0; j < 3; ++j) p[(12 + j) * stride] = vg.dS[j];
}
I3D_HD void voxel_deriv_park(const VoxelDeriv& vd, float* p, int stride)
{
#pragma unroll
    for (int i = 0; i < 4; ++i)
    {
#pragma unroll
        for (int k = 0; k < 3; ++k) { p[(3 * i + k) * stride] = vd.g[i][k]; p[(16 + 3 * i + k) * stride] = vd.A[i][k]; }
        p[(12 + i) * stride] = vd.il[i]; p[(28 + i) * stride] = vd.sigma[i]; p[(32 + i) * stride] = vd.s[i];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) p[(36 + k) * stride] = vd.X0[k];
    p[39 * stride] = vd.h;
}

// 1/x for the projection: MUFU seed + two Newton steps on the device (full double accuracy for normal x), plain division on the host
I3D_HD double rcp_f64(double a)
{
#ifdef __CUDA_ARCH__
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(a));
    r = fma(fma(-a, r, 1.0), r, r);
    r = fma(fma(-a, r, 1.0), r, r);
    // zero / inf / nan / denormal inputs: the seed is already the IEEE result or garbage-in-garbage-out; the row is invalid then
    return r;
#else
    return 1.0 / a;
#endif
}

template <bool DERIV>
I3D_HD void voxel_geom_make(const double sdf[10], const double alb[4], const int coord[3], double voxel_size, const double sh[9],
                            VoxelGeom* vg, VoxelDeriv* vd)
{
    double S[4];
    float shf[9];
    if (DERIV)
    {
#pragma unroll
        for (int k = 0; k < 9; ++k) shf[k] = static_cast<float>(sh[k]);
        vd->h = static_cast<float>(voxel_size);
#pragma unroll
        for (int k = 0; k < 3; ++k) vd->X0[k] = static_cast<float>(coord[k]) * vd->h;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
    {
        const double q0 = sdf[I3D_QUAD(i, 0)];
        double g[3] = {sdf[I3D_QUAD(i, 1)] - q0, sdf[I3D_QUAD(i, 2)] - q0, sdf[I3D_QUAD(i, 3)] - q0};
        const double len2 = g[0] * g[0] + g[1] * g[1] + g[2] * g[2];
        double il = 1.0;
        if (len2 > 0.0) { il = Num<double>::rsqrt_(len2); g[0] *= il; g[1] *= il; g[2] *= il; }
        const int c[3] = {coord[0] + (i == 1), coord[1] + (i == 2), coord[2] + (i == 3)};
#pragma unroll
        for (int k = 0; k < 3; ++k) vg->X[i][k] = static_cast<double>(c[k]) * voxel_size - g[k] * q0;
        S[i] = alb[i] * sh_eval<double>(sh, g, nullptr);
        if (DERIV)
        {
            const float gf[3] = {static_cast<float>(g[0]), static_cast<float>(g[1]), static_cast<float>(g[2])};
            float gs[3];
            vd->sigma[i] = sh_eval<float>(shf, gf, gs);
            const float af = static_cast<float>(alb[i]);
#pragma unroll
            for (int k = 0; k < 3; ++k) { vd->g[i][k] = gf[k]; vd->A[i][k] = af * gs[k]; }
            vd->il[i] = static_cast<float>(il);
            vd->s[i] = static_cast<float>(q0);
        }
    }
    vg->dS[0] = S[1] - S[0]; vg->dS[1] = S[2] - S[0]; vg->dS[2] = S[3] - S[0];
}

// Catmull-Rom weights of the four taps at fraction x (CubicHermiteSpline in weight form) and their derivatives
template <class T>
I3D_HD void cr_weights(T x, T w[4])
{
    const T x2 = x * x, x3 = x2 * x;
    w[0] = T(0.5) * (-x3 + T(2.0) * x2 - x);
    w[1] = T(0.5) * (T(3.0) * x3 - T(5.0) * x2 + T(2.0));
    w[2] = T(0.5) * (-T(3.0) * x3 + T(4.0) * x2 + x);
    w[3] = T(0.5) * (x3 - x2);
}
template <class T>
I3D_HD void cr_dweights(T x, T w[4])
{
    const T x2 = x * x;
    w[0] = T(0.5) * (-T(3.0) * x2 + T(4.0) * x - T(1.0));
    w[1] = T(0.5) * (T(9.0) * x2 - T(10.0) * x);
    w[2] = T(0.5) * (-T(9.0) * x2 + T(8.0) * x + T(1.0));
    w[3] = T(0.5) * (T(3.0) * x2 - T(2.0) * x);
}

// BiCubicInterpolator::Evaluate(r = v, c = u) on the clamped Grid2D<float>, split in three steps so that the taps of SEVERAL sample
// points can be in flight together (bicubic_locate all -> bicubic_taps all -> bicubic_eval all): value and (if GRAD) the image
// gradient (dL/du, dL/dv), all from the same 16 taps in double (the gradient is returned as float: it only feeds the float Jacobian).
// Evaluating the gradient in double costs fewer issue slots than a float evaluation that first has to subtract the centre tap to
// avoid the eps*|p|/|gradient| cancellation (a float gradient on the raw taps was 4e-5 off the oracle's Jets, tests/test_eg_math.py).
struct BicubicSite { int col, row; double xu, xv; };

// (w, h: image size.  A candidate state of a rejected / unfinished LM trial can project anywhere — or to NaN: the integer
// pixel is taken from the coordinate clamped to [-8, size + 8], which is the identity for every in-bounds row and keeps every index
// computation far from integer overflow; NaN coordinates still give NaN fractions, hence a non-finite residual = invalid row.)
I3D_HD void bicubic_locate(double u, double v, int w, int h, BicubicSite* s)
{
    const double fu = floor(fmin(fmax(u, -8.0), static_cast<double>(w) + 8.0)), fv = floor(fmin(fmax(v, -8.0), static_cast<double>(h) + 8.0));
    s->col = static_cast<int>(fu); s->row = static_cast<int>(fv);
    s->xu = u - fu; s->xv = v - fv;
}
I3D_HD bool bicubic_interior(const BicubicSite& s, int w, int h) { return s.col >= 1 && s.col + 2 <= w - 1 && s.row >= 1 && s.row + 2 <= h - 1; }

template <bool INTERIOR>
I3D_HD void bicubic_taps(const float* __restrict__ img, int w, int h, const BicubicSite& s, float p[16])
{
    if (INTERIOR)
    {
        const float* __restrict__ b = img + static_cast<size_t>(s.row - 1) * w + (s.col - 1);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j)
#ifdef __CUDA_ARCH__
                p[4 * i + j] = __ldg(b + static_cast<size_t>(i) * w + j);
#else
                p[4 * i + j] = b[static_cast<size_t>(i) * w + j];
#endif
    }
    else
    {
        int cc[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { int c = s.col - 1 + j; c = c < 0 ? 0 : c; cc[j] = c > w - 1 ? w - 1 : c; }
#pragma unroll
        for (int i = 0; i < 4; ++i)
        {
            int rr = s.row - 1 + i; rr = rr < 0 ? 0 : rr; rr = rr > h - 1 ? h - 1 : rr;
            const float* line = img + static_cast<size_t>(rr) * w;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#ifdef __CUDA_ARCH__
                p[4 * i + j] = __ldg(line + cc[j]);
#else
                p[4 * i + j] = line[cc[j]];
#endif
        }
    }
}

// Where the luminance taps of two sample points come from.  LinearImage: the frame as a pitch-linear float array (host harness and
// the fallback device path): 16 scalar loads per point, unclamped when both 4x4 neighbourhoods are interior.
struct LinearImage
{
    const float* __restrict__ img;
    I3D_HD void taps2(int w, int h, const BicubicSite& s0, const BicubicSite& s1, float p0[16], float p1[16]) const
    {
        if (bicubic_interior(s0, w, h) && bicubic_interior(s1, w, h))
        {
            bicubic_taps<true>(img, w, h, s0, p0);
            bicubic_taps<true>(img, w, h, s1, p1);
        }
        else
        {
            bicubic_taps<false>(img, w, h, s0, p0);
            bicubic_taps<false>(img, w, h, s1, p1);
        }
    }
};

// (Measured dead end, round 2: the frames as 2D CUDA arrays behind per-frame texture objects, a 4x4 neighbourhood fetched with four
// tld4 gathers under clamp addressing — bit-exact, but 5x SLOWER (k_eg_rows 3.9 ms vs 0.73 ms at C3): the lanes of a warp select
// different frames, i.e. different bindless texture headers, and the gather serialises per distinct header.)

template <bool GRAD>
I3D_HD double bicubic_eval(const BicubicSite& s, const float p[16], float* Lu, float* Lv)
{
    double wu[4], wv[4], du[4], dv[4];
    cr_weights<double>(s.xu, wu);
    cr_weights<double>(s.xv, wv);
    if (GRAD) { cr_dweights<double>(s.xu, du); cr_dweights<double>(s.xv, dv); }
    double L = 0.0, lu = 0.0, lv = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
    {
        const double p0 = static_cast<double>(p[4 * i]), p1 = static_cast<double>(p[4 * i + 1]), p2 = static_cast<double>(p[4 * i + 2]), p3 = static_cast<double>(p[4 * i + 3]);
        const double ri = fma(wu[0], p0, fma(wu[1], p1, fma(wu[2], p2, wu[3] * p3)));
        L = fma(wv[i], ri, L);
        if (GRAD)
        {
            const double rd = fma(du[0], p0, fma(du[1], p1, fma(du[2], p2, du[3] * p3)));
            lu = fma(wv[i], rd, lu);
            lv = fma(dv[i], ri, lv);
        }
    }
    if (GRAD) { *Lu = static_cast<float>(lu); *Lv = static_cast<float>(lv); }
    return L;
}

// what the derivative pass needs from the primal of one sample point
struct PointSave { float x, y, iz, Lu, Lv; };

// Primal of one row: the four per-frame projections + luminance lookups.  Returns the residual (0.0 = invalid row).
// e[4] (if DERIV and the row is valid and non-zero): d r / d (S_i - L_i) = (-(sum), d1, d2, d3) / r.
template <bool DERIV, class VG, class IMG>
I3D_HD double eg_frame_primal(const VG& vg, const FramePose& fp, const CamParams<double>& cam, const IMG& img,
                              PointSave sv[4], float e[4])
{
    // phase 1: the four projections (float64 chains, independent of each other and of any luminance load)
    double u[4], v[4];
    bool inb = true;
#pragma unroll
    for (int i = 0; i < 4; ++i)
    {
        const double X0 = vg.Xv(i, 0), X1 = vg.Xv(i, 1), X2 = vg.Xv(i, 2);
        const double Y0 = fp.R[0] * X0 + fp.R[1] * X1 + fp.R[2] * X2 + fp.t[0];
        const double Y1 = fp.R[3] * X0 + fp.R[4] * X1 + fp.R[5] * X2 + fp.t[1];
        const double Y2 = fp.R[6] * X0 + fp.R[7] * X1 + fp.R[8] * X2 + fp.t[2];
        const double iz = rcp_f64(Y2);
        const double x = Y0 * iz, y = Y1 * iz;
        const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
        const double dc = 1.0 + cam.k1 * r2 + cam.k2 * r4 + cam.k3 * r6;
        const double xd = x * dc + 2.0 * cam.p1 * x * y + cam.p2 * (r2 + 2.0 * x * x);
        const double yd = y * dc + 2.0 * cam.p2 * xd * y + cam.p1 * (r2 + 2.0 * y * y);
        u[i] = cam.fx * xd + cam.cx; v[i] = cam.fy * yd + cam.cy;
        // same comparison as CameraT::project (NaN => comparisons false => "inside", caught by the finite test below)
        if (u[i] < 0.0 || u[i] > static_cast<double>(cam.w - 1) || v[i] < 0.0 || v[i] > static_cast<double>(cam.h - 1)) inb = false;
        if (DERIV) { sv[i].x = static_cast<float>(x); sv[i].y = static_cast<float>(y); sv[i].iz = static_cast<float>(iz); }
    }
    // phase 2: the bicubic lookups, two points at a time: the 32 taps of a pair are issued back to back (one basic block when both
    // 4x4 neighbourhoods are interior), so their L1/L2 latencies overlap instead of being paid once per point
    double L[4];
#pragma unroll
    for (int i = 0; i < 4; i += 2)
    {
        BicubicSite s0, s1;
        bicubic_locate(u[i], v[i], cam.w, cam.h, &s0);
        bicubic_locate(u[i + 1], v[i + 1], cam.w, cam.h, &s1);
        float p0[16], p1[16];
        img.taps2(cam.w, cam.h, s0, s1, p0, p1);
        float lu = 0.0f, lv = 0.0f;
        L[i] = bicubic_eval<DERIV>(s0, p0, &lu, &lv);
        if (DERIV) { sv[i].Lu = lu; sv[i].Lv = lv; }
        L[i + 1] = bicubic_eval<DERIV>(s1, p1, &lu, &lv);
        if (DERIV) { sv[i + 1].Lu = lu; sv[i + 1].Lv = lv; }
    }
    if (!inb) return 0.0;
    const double d1 = vg.dSv(0) - (L[1] - L[0]);
    const double d2 = vg.dSv(1) - (L[2] - L[0]);
    const double d3 = vg.dSv(2) - (L[3] - L[0]);
    const double r = sqrt(d1 * d1 + d2 * d2 + d3 * d3);
    if (!finite_(r)) return 0.0;
    if (DERIV && r != 0.0)
    {
        const double ir = 1.0 / r;
        e[0] = static_cast<float>(-(d1 + d2 + d3) * ir); e[1] = static_cast<float>(d1 * ir); e[2] = static_cast<float>(d2 * ir); e[3] = static_cast<float>(d3 * ir);
    }
    return r;
}

// Derivative of one valid row (float): fills row[29].
template <class VD>
I3D_HD void eg_frame_deriv(const VD& vd, const FramePose& fp, const CamParams<float>& cam, const PointSave sv[4], const float e[4],
                           float* __restrict__ row)
{
#pragma unroll
    for (int k = 0; k < 29; ++k) row[k] = 0.0f;
    float m[3] = {0.0f, 0.0f, 0.0f};      // sum_i e_i X_i x (R^T dL/dY_i)
    float tacc[3] = {0.0f, 0.0f, 0.0f};   // sum_i e_i dL/dY_i
#define I3D_POINT_DERIV(POINT)                                                                                                        \
    {                                                                                                                                 \
        const int i = POINT;                                                                                                          \
        const float x = sv[i].x, y = sv[i].y, iz = sv[i].iz, Lu = sv[i].Lu, Lv = sv[i].Lv, ei = e[i];                                 \
        const float r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;                                                                   \
        const float dc = 1.0f + cam.k1 * r2 + cam.k2 * r4 + cam.k3 * r6;                                                              \
        const float dcp = cam.k1 + 2.0f * cam.k2 * r2 + 3.0f * cam.k3 * r4;                                                           \
        const float xd = x * dc + 2.0f * cam.p1 * x * y + cam.p2 * (r2 + 2.0f * x * x);                                               \
        const float yd = y * dc + 2.0f * cam.p2 * xd * y + cam.p1 * (r2 + 2.0f * y * y);                                              \
        const float xdx = dc + 2.0f * x * x * dcp + 2.0f * cam.p1 * y + 6.0f * cam.p2 * x;                                            \
        const float xdy = 2.0f * x * y * dcp + 2.0f * cam.p1 * x + 2.0f * cam.p2 * y;                                                 \
        const float ydx = 2.0f * x * y * dcp + 2.0f * cam.p2 * y * xdx + 2.0f * cam.p1 * x;                                           \
        const float ydy = dc + 2.0f * y * y * dcp + 2.0f * cam.p2 * (y * xdy + xd) + 6.0f * cam.p1 * y;                              \
        const float gu = Lu * cam.fx, gv = Lv * cam.fy;                                                                               \
        const float Lx = gu * xdx + gv * ydx, Ly = gu * xdy + gv * ydy;                                                               \
        const float LY0 = Lx * iz, LY1 = Ly * iz, LY2 = -(Lx * x + Ly * y) * iz;                                                      \
        const float LX0 = LY0 * fp.Rf[0] + LY1 * fp.Rf[3] + LY2 * fp.Rf[6];                                                           \
        const float LX1 = LY0 * fp.Rf[1] + LY1 * fp.Rf[4] + LY2 * fp.Rf[7];                                                           \
        const float LX2 = LY0 * fp.Rf[2] + LY1 * fp.Rf[5] + LY2 * fp.Rf[8];                                                           \
        const float s = vd.sv(i), g0 = vd.gv(i, 0), g1 = vd.gv(i, 1), g2 = vd.gv(i, 2);                                              \
        const float Xf0 = vd.X0v(0) + (i == 1 ? vd.hv() : 0.0f) - g0 * s;                                                            \
        const float Xf1 = vd.X0v(1) + (i == 2 ? vd.hv() : 0.0f) - g1 * s;                                                            \
        const float Xf2 = vd.X0v(2) + (i == 3 ? vd.hv() : 0.0f) - g2 * s;                                                            \
        const float c0 = fp.small ? LY0 : LX0, c1 = fp.small ? LY1 : LX1, c2 = fp.small ? LY2 : LX2;                                  \
        m[0] += ei * (Xf1 * c2 - Xf2 * c1); m[1] += ei * (Xf2 * c0 - Xf0 * c2); m[2] += ei * (Xf0 * c1 - Xf1 * c0);                   \
        tacc[0] += ei * LY0; tacc[1] += ei * LY1; tacc[2] += ei * LY2;                                                                \
        row[20] -= ei * (Lu * cam.pyr_scale * xd);                                                                                    \
        row[21] -= ei * (Lv * cam.pyr_scale * yd);                                                                                    \
        row[22] -= ei * (Lu * cam.pyr_scale);                                                                                         \
        row[23] -= ei * (Lv * cam.pyr_scale);                                                                                         \
        {                                                                                                                             \
            const float c2y = 2.0f * cam.p2 * y;                                                                                      \
            const float xk1 = x * r2, xk2 = x * r4, xk3 = x * r6, xp1 = 2.0f * x * y, xp2 = r2 + 2.0f * x * x;                        \
            row[24] -= ei * (gu * xk1 + gv * (y * r2 + c2y * xk1));                                                                   \
            row[25] -= ei * (gu * xk2 + gv * (y * r4 + c2y * xk2));                                                                   \
            row[26] -= ei * (gu * xk3 + gv * (y * r6 + c2y * xk3));                                                                   \
            row[27] -= ei * (gu * xp1 + gv * ((r2 + 2.0f * y * y) + c2y * xp1));                                                      \
            row[28] -= ei * (gu * xp2 + gv * (2.0f * xd * y + c2y * xp2));                                                            \
        }                                                                                                                             \
        const float vn0 = vd.Av(i, 0) + s * LX0, vn1 = vd.Av(i, 1) + s * LX1, vn2 = vd.Av(i, 2) + s * LX2;                         \
        const float gd = g0 * vn0 + g1 * vn1 + g2 * vn2;                                                                              \
        const float il = vd.ilv(i);                                                                                                   \
        const float d1 = il * (vn0 - g0 * gd), d2 = il * (vn1 - g1 * gd), d3 = il * (vn2 - g2 * gd);                                  \
        const float d0 = -(d1 + d2 + d3) + (g0 * LX0 + g1 * LX1 + g2 * LX2);                                                          \
        row[I3D_QUAD(POINT, 0)] += ei * d0;                                                                                           \
        row[I3D_QUAD(POINT, 1)] += ei * d1;                                                                                           \
        row[I3D_QUAD(POINT, 2)] += ei * d2;                                                                                           \
        row[I3D_QUAD(POINT, 3)] += ei * d3;                                                                                           \
        row[10 + POINT] += ei * vd.sigmav(i);                                                                                        \
    }
    I3D_POINT_DERIV(0)
    I3D_POINT_DERIV(1)
    I3D_POINT_DERIV(2)
    I3D_POINT_DERIV(3)
#undef I3D_POINT_DERIV
#pragma unroll
    for (int c = 0; c < 3; ++c)
    {
        row[14 + c] = -(m[0] * fp.Jr[c] + m[1] * fp.Jr[3 + c] + m[2] * fp.Jr[6 + c]);
        row[17 + c] = -tacc[c];
    }
}

} // namespace i3d
