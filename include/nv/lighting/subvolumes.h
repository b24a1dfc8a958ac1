// nv/lighting/subvolumes.h — Subvolumes with the reference's query API (libintrinsic3d/include/nv/lighting/subvolumes.h:47-90),
// filled from the H100 engine's subvolume table (i3d_download_lighting) instead of a host pass over the hash.
//
// Numbering: ascending (z, y, x) of the integer cube index (the reference numbers in std::unordered_map iteration order, which
// is unspecified; nothing downstream depends on it).  bounds()/color() exist for API completeness (debug visualisation only).
#pragma once
#include <cmath>
#include <unordered_map>
#include <vector>

#include <nv/mat.h>
#include <nv/sparse_voxel_grid.h>

namespace nv
{
using Vec6i = VecN<int, 6>;

class Subvolumes
{
public:
    explicit Subvolumes(float size) : size_(size) {}

    void clear() { subvolumes_.clear(); indices_.clear(); }
    // Subvolumes::compute(grid) of the reference; here the table comes from the device (LightingSVSH::estimate calls it)
    void assign(float voxel_size, const std::vector<int32_t>& index3)
    {
        clear();
        voxel_size_ = voxel_size;
        for (size_t i = 0; i + 2 < index3.size(); i += 3)
        {
            const Vec3i idx{index3[i], index3[i + 1], index3[i + 2]};
            subvolumes_[idx] = static_cast<int>(indices_.size());
            indices_.push_back(idx);
        }
    }

    float subvolumeSize() const { return size_; }
    size_t count() const { return indices_.size(); }
    Vec3i index(int subvol) const { return indices_[static_cast<size_t>(subvol)]; }
    Vec6i bounds(int subvol) const
    {
        const Vec3i idx = index(subvol);
        Vec6i b;
        for (int d = 0; d < 3; ++d) { b[2 * d] = indexToVoxel(idx[d]); b[2 * d + 1] = indexToVoxel(idx[d] + 1) - 1; }
        return b;
    }
    bool exists(int subvol) const { return subvol >= 0 && subvol < static_cast<int>(indices_.size()); }
    bool exists(const Vec3i& idx) const { return exists(indexToSubvolume(idx)); }
    Vec3f pointToIndexCoord(const Vec3f& pt) const
    {
        Vec3f r;
        for (int d = 0; d < 3; ++d) r[d] = pt[d] * (1.0f / size_) - 0.5f;
        return r;
    }
    int pointToSubvolume(const Vec3f& p) const
    {
        Vec3i idx;
        for (int d = 0; d < 3; ++d) idx[d] = static_cast<int>(std::floor(p[d] * (1.0f / size_)));
        return indexToSubvolume(idx);
    }
    int indexToSubvolume(const Vec3i& idx) const
    {
        auto it = subvolumes_.find(idx);
        return it == subvolumes_.end() ? -1 : it->second;
    }
    // trilinear blend of per-subvolume 9-vectors at a world point (Subvolumes::interpolate<Eigen::VectorXd>, linear = true)
    VecXd interpolate(const std::vector<VecXd>& values, const Vec3f& pt, bool linear = true) const;

private:
    int indexToVoxel(int idx) const { return static_cast<int>(std::round(static_cast<float>(idx) * size_ / voxel_size_)); }

    float size_;
    float voxel_size_ = 0.0f;
    std::unordered_map<Vec3i, int> subvolumes_;
    std::vector<Vec3i> indices_;
};
} // namespace nv
