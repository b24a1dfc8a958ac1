/*
 * i3d_grid.cuh — what every device module of the engine shares about the grid: the neighbour-table slots, the block size, the device
 * hash (coordinates -> voxel index) and the explicitly rounded float operations.  No kernels: i3d_kernels.cuh (the engine's module)
 * and i3d_mesh.cuh (the surface extraction's module) both include it.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace i3d
{

// neighbour-table slots
enum { NB_XP = 0, NB_XM, NB_YP, NB_YM, NB_ZP, NB_ZM, NB_X2, NB_Y2, NB_Z2, NB_XY, NB_XZ, NB_YZ, NB_COUNT };

constexpr int kThreads = 256;

// ----------------------------------------------------------------------------------------------
// exact float arithmetic (no FMA contraction): must round like oracle.cpp / the reference's float code
// ----------------------------------------------------------------------------------------------
#define FM(a, b) __fmul_rn((a), (b))
#define FA(a, b) __fadd_rn((a), (b))
#define FS(a, b) __fsub_rn((a), (b))
#define FD(a, b) __fdiv_rn((a), (b))

// ----------------------------------------------------------------------------------------------
// device hash table of the grid (replaces unordered_map::find, sparse_voxel_grid.cpp:166-259)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t pack_key(int x, int y, int z)
{
    return ((static_cast<uint64_t>(x + (1 << 20)) & 0x1FFFFFull) << 42) | ((static_cast<uint64_t>(y + (1 << 20)) & 0x1FFFFFull) << 21) |
           (static_cast<uint64_t>(z + (1 << 20)) & 0x1FFFFFull);
}
__device__ __forceinline__ uint64_t mix64(uint64_t k)
{
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return k;
}
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;

// (noinline: runs once per grid upload; keeps the 12 probe loops out of the caller.  inline: one definition per translation unit)
inline __device__ __noinline__ int32_t hash_find(const unsigned long long* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask, int x, int y, int z)
{
    const unsigned long long key = pack_key(x, y, z);
    uint64_t slot = mix64(key) & mask;
    while (true)
    {
        const unsigned long long k = keys[slot];
        if (k == key) return vals[slot];
        if (k == kEmptyKey) return -1;
        slot = (slot + 1) & mask;
    }
}

} // namespace i3d
