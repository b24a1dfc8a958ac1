/*
 * i3d_fusion_view.cuh — the fusion volume in progress as a reader sees it: the slot values of the fusion's hash table, a read-only view of
 * its table and Voxel arrays, and the probe.  No kernels: the fusion module (i3d_fusion.cuh) and the tracker's prediction from the volume
 * in progress (i3d_render.cuh) both include it, so the slot layout is written down once.
 */
#pragma once
#include "i3d_grid.cuh"

namespace i3d
{

// hash value of the fusion table: voxel index in the low 31 bits, bit 31 = "the 3x3x3 block around this voxel is complete"
constexpr unsigned kFuseBlockBit = 0x80000000u;
constexpr unsigned kFuseIndexMask = 0x7FFFFFFFu;

// The volume in progress, read-only: table keys / vals with mask = slots - 1, and the Voxel {sdf, weight} arrays of the n allocated
// voxels with their coordinates, indexed [0, n) in slot-claim order
struct FuseView
{
    const unsigned long long* keys; const unsigned* vals; uint64_t mask;
    const int32_t* x; const int32_t* y; const int32_t* z;
    const float* sdf; const float* weight;
    int64_t n;
};

// The voxel index of (x, y, z) in the fusion table, or -1
__device__ __forceinline__ int32_t fuse_find(const unsigned long long* __restrict__ keys, const unsigned* __restrict__ vals, uint64_t mask, int x, int y, int z)
{
    const unsigned long long key = pack_key(x, y, z);
    uint64_t slot = mix64(key) & mask;
    while (true)
    {
        const unsigned long long k = keys[slot];
        if (k == key) return static_cast<int32_t>(vals[slot] & kFuseIndexMask);
        if (k == kEmptyKey) return -1;
        slot = (slot + 1) & mask;
    }
}

} // namespace i3d
