/*
 * check_cull.cu — test harness of the conservative frame culling of the frame scans (i3d_observe.cuh), not part of the product library.
 *
 * For every (sphere, frame) case it evaluates frame_may_see on the depth tiles that k_depth_tiles builds, and probes points of the
 * sphere with the exact observation weight of the frame scans (obs_probe + obs_finish): the centre, the 6 axis extremes, the points
 * nearest to and farthest from the camera centre, and n_random seeded interior points.  The normal of each probe faces the camera, so
 * a probe that passes the reference's image, depth and occlusion tests has weight > 0.  A case with frame_may_see == false and a probe
 * of weight > 0 is a frame the culling would drop although the reference observes it.  Everything is called from the engine's headers;
 * nothing is restated here.  tests/test_gpu_zz_cull_bound.py drives it.
 */
#include "../../intrinsic3d_b200/csrc/i3d_kernels.cuh"

#include <cuda_runtime.h>
#include <stdint.h>

using namespace i3d;

namespace
{

__device__ __forceinline__ uint64_t splitmix(uint64_t& s)
{
    uint64_t z = (s += 0x9e3779b97f4a7c15ull);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ float unit(uint64_t& s) { return static_cast<float>(splitmix(s) >> 40) * (1.0f / 16777216.0f); }   // [0, 1)

// cams: per frame fx, fy, cx, cy, d[0..4] = k1, k2, k3, p1, p2 (SelectCam's order), occlusion
__global__ void k_check(int F, int W, int H, const float* __restrict__ depth, const float* __restrict__ rt, const float* __restrict__ cams,
                        const float* __restrict__ tmin, const float* __restrict__ tmax, int S, const float* __restrict__ sph,
                        const int32_t* __restrict__ sph_frame, int n_random, uint64_t seed, uint8_t* __restrict__ may, int32_t* __restrict__ hits,
                        float* __restrict__ hit_pt)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const int f = sph_frame[s];
    const float* Rt = rt + 12 * f;
    const float* cp = cams + 10 * f;
    SelectCam cam;
    cam.fx = cp[0]; cam.fy = cp[1]; cam.cx = cp[2]; cam.cy = cp[3];
    cam.dist_zero = 1;
    for (int k = 0; k < 5; ++k) { cam.d[k] = cp[4 + k]; if (cam.d[k] != 0.0f) cam.dist_zero = 0; }
    cam.occlusion = cp[9];
    const CullView cv{tmin, tmax, 1, nullptr};
    const float c[3] = {sph[4 * s], sph[4 * s + 1], sph[4 * s + 2]};
    const float rad = sph[4 * s + 3];
    may[s] = frame_may_see(c, rad, Rt, cam, cv, f, W, H) ? 1 : 0;
    // camera centre -R^T t: the direction of the nearest point and the normal that faces the camera
    float cc[3];
    for (int k = 0; k < 3; ++k) cc[k] = -(Rt[k] * Rt[9] + Rt[3 + k] * Rt[10] + Rt[6 + k] * Rt[11]);
    float toc[3] = {cc[0] - c[0], cc[1] - c[1], cc[2] - c[2]};
    float l = sqrtf(toc[0] * toc[0] + toc[1] * toc[1] + toc[2] * toc[2]);
    if (!(l > 0.0f)) { toc[0] = 0.0f; toc[1] = 0.0f; toc[2] = 1.0f; l = 1.0f; }
    for (int k = 0; k < 3; ++k) toc[k] /= l;
    const float* img = depth + static_cast<size_t>(f) * W * H;
    uint64_t st = seed ^ (0x5851f42d4c957f2dull * static_cast<uint64_t>(s + 1));
    int nhit = 0;
    const int nprobe = 9 + n_random;
    for (int i = 0; i < nprobe; ++i)
    {
        float u[3] = {0.0f, 0.0f, 0.0f};
        if (i >= 1 && i <= 6) u[(i - 1) >> 1] = (i & 1) ? 1.0f : -1.0f;
        else if (i == 7) { u[0] = toc[0]; u[1] = toc[1]; u[2] = toc[2]; }
        else if (i == 8) { u[0] = -toc[0]; u[1] = -toc[1]; u[2] = -toc[2]; }
        else if (i > 8)
        {
            // uniform in the ball: a direction (rejection in the cube) and radius cbrt(U); every 4th point on the sphere's surface
            float n2;
            do { for (int k = 0; k < 3; ++k) u[k] = 2.0f * unit(st) - 1.0f; n2 = u[0] * u[0] + u[1] * u[1] + u[2] * u[2]; } while (n2 > 1.0f || n2 < 1e-6f);
            const float r = ((i & 3) == 0) ? 1.0f : cbrtf(unit(st));
            const float sc = r * rsqrtf(n2);
            for (int k = 0; k < 3; ++k) u[k] *= sc;
        }
        const float pt[3] = {c[0] + rad * u[0], c[1] + rad * u[1], c[2] + rad * u[2]};
        float nrm[3] = {cc[0] - pt[0], cc[1] - pt[1], cc[2] - pt[2]};
        const float nl = sqrtf(nrm[0] * nrm[0] + nrm[1] * nrm[1] + nrm[2] * nrm[2]);
        if (nl > 0.0f && isfinite(nl)) for (int k = 0; k < 3; ++k) nrm[k] /= nl;
        else { nrm[0] = 0.0f; nrm[1] = 0.0f; nrm[2] = 1.0f; }
        const float w = obs_finish(obs_probe(pt, Rt, cam, img, W, H), nrm, Rt, cam);
        if (w > 0.0f)
        {
            if (nhit == 0) { hit_pt[3 * s] = pt[0]; hit_pt[3 * s + 1] = pt[1]; hit_pt[3 * s + 2] = pt[2]; }
            ++nhit;
        }
    }
    hits[s] = nhit;
}

template <class T>
int dev_copy(T** d, const T* h, size_t n)
{
    if (cudaMalloc(d, n * sizeof(T) + 16) != cudaSuccess) return 1;
    return h && cudaMemcpy(*d, h, n * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess;
}

} // namespace

// Returns 0 on success, else a CUDA error code.  tiles (optional): the [2][F][TH][TW] tile minima and maxima, for the test's own checks.
extern "C" int check_cull(int F, int W, int H, const float* depth, const float* rt, const float* cams, int S, const float* sph,
                          const int32_t* sph_frame, int n_random, uint64_t seed, uint8_t* may, int32_t* hits, float* hit_pt, float* tiles)
{
    const int TW = (W + kCullTile - 1) / kCullTile, TH = (H + kCullTile - 1) / kCullTile;
    const size_t nt = static_cast<size_t>(F) * TW * TH;
    float *d_depth = nullptr, *d_rt = nullptr, *d_cams = nullptr, *d_sph = nullptr, *d_tmin = nullptr, *d_tmax = nullptr, *d_pt = nullptr;
    int32_t *d_frame = nullptr, *d_hits = nullptr;
    uint8_t* d_may = nullptr;
    int bad = dev_copy(&d_depth, depth, static_cast<size_t>(F) * W * H) | dev_copy(&d_rt, rt, 12 * static_cast<size_t>(F)) |
              dev_copy(&d_cams, cams, 10 * static_cast<size_t>(F)) | dev_copy(&d_sph, sph, 4 * static_cast<size_t>(S)) |
              dev_copy(&d_frame, sph_frame, static_cast<size_t>(S)) | dev_copy<float>(&d_tmin, nullptr, nt) | dev_copy<float>(&d_tmax, nullptr, nt) |
              dev_copy<float>(&d_pt, nullptr, 3 * static_cast<size_t>(S)) | dev_copy<int32_t>(&d_hits, nullptr, S) | dev_copy<uint8_t>(&d_may, nullptr, S);
    cudaError_t err = bad ? cudaErrorMemoryAllocation : cudaMemset(d_pt, 0xff, 3 * static_cast<size_t>(S) * sizeof(float));   // NaN: no hit
    if (err == cudaSuccess)
    {
        // the engine's launch (install_frames)
        k_depth_tiles<<<static_cast<unsigned>(nt), 256>>>(F, W, H, d_depth, d_tmin, d_tmax);
        k_check<<<(S + 127) / 128, 128>>>(F, W, H, d_depth, d_rt, d_cams, d_tmin, d_tmax, S, d_sph, d_frame, n_random, seed, d_may, d_hits, d_pt);
        err = cudaDeviceSynchronize();
    }
    if (err == cudaSuccess) err = cudaMemcpy(may, d_may, S, cudaMemcpyDeviceToHost);
    if (err == cudaSuccess) err = cudaMemcpy(hits, d_hits, S * sizeof(int32_t), cudaMemcpyDeviceToHost);
    if (err == cudaSuccess) err = cudaMemcpy(hit_pt, d_pt, 3 * static_cast<size_t>(S) * sizeof(float), cudaMemcpyDeviceToHost);
    if (err == cudaSuccess && tiles) err = cudaMemcpy(tiles, d_tmin, nt * sizeof(float), cudaMemcpyDeviceToHost);
    if (err == cudaSuccess && tiles) err = cudaMemcpy(tiles + nt, d_tmax, nt * sizeof(float), cudaMemcpyDeviceToHost);
    void* bufs[] = {d_depth, d_rt, d_cams, d_sph, d_tmin, d_tmax, d_pt, d_frame, d_hits, d_may};
    for (void* b : bufs) cudaFree(b);
    return static_cast<int>(err);
}
