// nv/rgbd/pyramid.h — per-keyframe image pyramid as the optimiser sees it (reference: include/nv/rgbd/pyramid.h:47-69).
// The caller attaches float luminance and depth images per level.  A pyramid that carries only level 0 and its colour image is
// enough for Intrinsic3D::refine: the engine then builds the coarser levels on the device (Pyramid::create's pyrDown and
// downsampleDepth chains, i3d_use_rgbd_level; DESIGN.md §6i).
#pragma once
#include <vector>

#include <nv/image.h>

namespace nv
{
class Pyramid
{
public:
    void addLevel(const ImageF& intensity, const ImageF& depth) { intensity_.push_back(intensity); depth_.push_back(depth); color_.push_back(ImageBGR()); }
    void addLevel(const ImageF& intensity, const ImageF& depth, const ImageBGR& color) { intensity_.push_back(intensity); depth_.push_back(depth); color_.push_back(color); }
    int levels() const { return static_cast<int>(intensity_.size()); }
    ImageF intensity(int lvl) const { return intensity_[static_cast<size_t>(lvl)]; }
    ImageF depth(int lvl) const { return depth_[static_cast<size_t>(lvl)]; }
    ImageBGR color(int lvl) const { return color_[static_cast<size_t>(lvl)]; }

private:
    std::vector<ImageF> intensity_, depth_;
    std::vector<ImageBGR> color_;
};
} // namespace nv
