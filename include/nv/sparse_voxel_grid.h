// nv/sparse_voxel_grid.h — API-shaped stand-in for the reference's voxel hash
// (libintrinsic3d/include/nv/sparse_voxel_grid.h:69-161, src/sparse_voxel_grid.cpp:166-259).
// Only what the refinement path touches is provided: VoxelSBR, iteration, exists/valid/voxel, voxelSize, truncation.
// Iteration order is insertion order (deterministic); it defines the "voxel_idx" the engine uses.
#pragma once
#include <cstdint>
#include <cstring>
#include <fstream>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include <nv/mat.h>

namespace nv
{
// basic voxel of the fused TSDF (include/nv/sparse_voxel_grid.h:56-62); the .tsdf files hold these
struct Voxel
{
    float sdf = 0.0f;
    float weight = 0.0f;
    Vec3b color = Vec3b::Zero();
};

struct VoxelSBR
{
    double sdf = 0.0;
    float weight = 0.0f;
    Vec3b color = Vec3b::Zero();
    double albedo = 0.6;
    double sdf_refined = 0.0;
};

template <class T>
class SparseVoxelGrid
{
public:
    using value_type = std::pair<Vec3i, T>;
    using iterator = typename std::vector<value_type>::iterator;
    using const_iterator = typename std::vector<value_type>::const_iterator;

    static SparseVoxelGrid* create(float voxel_size, float depth_min = 0.1f, float depth_max = 10.0f)
    {
        (void)depth_min; (void)depth_max;
        auto* g = new SparseVoxelGrid();
        g->voxel_size_ = voxel_size;
        g->truncation_ = voxel_size * 5.0f;
        return g;
    }
    iterator begin() { return nodes_.begin(); }
    iterator end() { return nodes_.end(); }
    const_iterator begin() const { return nodes_.begin(); }
    const_iterator end() const { return nodes_.end(); }
    bool empty() const { return nodes_.empty(); }
    size_t numVoxels() const { return nodes_.size(); }
    float voxelSize() const { return voxel_size_; }
    float truncation() const { return truncation_; }

    bool exists(const Vec3i& p) const { return index_.find(p) != index_.end(); }
    bool exists(int x, int y, int z) const { return exists(Vec3i{x, y, z}); }
    bool valid(const Vec3i& p) const { auto it = index_.find(p); return it != index_.end() && nodes_[it->second].second.weight > 0.0f; }
    bool valid(int x, int y, int z) const { return valid(Vec3i{x, y, z}); }
    T& voxel(const Vec3i& p) { return nodes_[index_.find(p)->second].second; }
    const T& voxel(const Vec3i& p) const { return nodes_[index_.find(p)->second].second; }
    T& voxel(int x, int y, int z) { return voxel(Vec3i{x, y, z}); }
    // insertion (the reference fills the grid by TSDF fusion / file load; fusion runs on the device, i3d_fusion_* in i3d_c_api.h)
    T& insert(const Vec3i& p, const T& v = T())
    {
        auto it = index_.find(p);
        if (it != index_.end()) { nodes_[it->second].second = v; return nodes_[it->second].second; }
        index_.emplace(p, nodes_.size());
        nodes_.emplace_back(p, v);
        return nodes_.back().second;
    }
    void reserve(size_t n) { nodes_.reserve(n); index_.reserve(n * 2); }
    void clear() { nodes_.clear(); index_.clear(); }
    float depthMin() const { return 0.1f; }
    float depthMax() const { return 10.0f; }

    // .tsdf files (src/sparse_voxel_grid.cpp:484-549): float voxel_size, truncation, integration_weight_sample; size_t count; float
    // max_load_factor; then per voxel the raw Vec3i (12 bytes) followed by the raw voxel struct (Voxel: 12 bytes, VoxelSBR: 32 bytes,
    // the reference's in-memory layout on x86-64).  Records are written in iteration order; padding bytes are zero.
    bool save(const std::string& filename) const
    {
        if (filename.empty()) return false;
        std::ofstream out(filename, std::ios::binary);
        if (!out.is_open()) return false;
        // header values of the loaded file are written back unchanged (defaults = the reference's constants, sparse_voxel_grid.cpp:49-53)
        const float integration_weight_sample = integration_weight_sample_, max_load_factor = max_load_factor_;
        const uint64_t size = nodes_.size();
        out.write(reinterpret_cast<const char*>(&voxel_size_), sizeof(float));
        out.write(reinterpret_cast<const char*>(&truncation_), sizeof(float));
        out.write(reinterpret_cast<const char*>(&integration_weight_sample), sizeof(float));
        out.write(reinterpret_cast<const char*>(&size), sizeof(uint64_t));
        out.write(reinterpret_cast<const char*>(&max_load_factor), sizeof(float));
        for (const auto& kv : nodes_)
        {
            char rec[12 + sizeof(T)];
            std::memset(rec, 0, sizeof(rec));
            const int32_t c[3] = {kv.first[0], kv.first[1], kv.first[2]};
            std::memcpy(rec, c, 12);
            voxelToBytes(kv.second, rec + 12);
            out.write(rec, sizeof(rec));
        }
        return out.good();
    }
    bool load(const std::string& filename)
    {
        if (filename.empty()) return false;
        clear();
        std::ifstream in(filename, std::ios::binary);
        if (!in.is_open()) return false;
        float integration_weight_sample = 0.0f, max_load_factor = 0.0f;
        uint64_t size = 0;
        in.read(reinterpret_cast<char*>(&voxel_size_), sizeof(float));
        in.read(reinterpret_cast<char*>(&truncation_), sizeof(float));
        in.read(reinterpret_cast<char*>(&integration_weight_sample), sizeof(float));
        in.read(reinterpret_cast<char*>(&size), sizeof(uint64_t));
        in.read(reinterpret_cast<char*>(&max_load_factor), sizeof(float));
        if (!in.good()) return false;
        // a corrupt / truncated header must not turn into a huge allocation: the count is bounded by what the file can hold
        {
            const std::streampos here = in.tellg();
            in.seekg(0, std::ios::end);
            const std::streampos end = in.tellg();
            in.seekg(here);
            const uint64_t room = (end > here) ? static_cast<uint64_t>(end - here) / (12 + sizeof(T)) : 0;
            if (size > room) return false;
        }
        integration_weight_sample_ = integration_weight_sample; max_load_factor_ = max_load_factor;
        reserve(static_cast<size_t>(size));
        for (uint64_t i = 0; i < size; ++i)
        {
            char rec[12 + sizeof(T)];
            in.read(rec, sizeof(rec));
            if (!in.good()) { clear(); return false; }          // the reference asserts; a truncated file is an error here
            int32_t c[3];
            std::memcpy(c, rec, 12);
            T v;
            voxelFromBytes(rec + 12, v);
            insert(Vec3i{c[0], c[1], c[2]}, v);
        }
        return true;
    }
    void setVoxel(const Vec3i& p, const T& v) { insert(p, v); }

private:
    // field-wise (de)serialisation at the offsets of the reference's structs
    static void voxelToBytes(const Voxel& v, char* b) { std::memcpy(b, &v.sdf, 4); std::memcpy(b + 4, &v.weight, 4); std::memcpy(b + 8, v.color.data(), 3); }
    static void voxelFromBytes(const char* b, Voxel& v) { std::memcpy(&v.sdf, b, 4); std::memcpy(&v.weight, b + 4, 4); std::memcpy(v.color.data(), b + 8, 3); }
    static void voxelToBytes(const VoxelSBR& v, char* b)
    {
        std::memcpy(b, &v.sdf, 8); std::memcpy(b + 8, &v.weight, 4); std::memcpy(b + 12, v.color.data(), 3); std::memcpy(b + 16, &v.albedo, 8); std::memcpy(b + 24, &v.sdf_refined, 8);
    }
    static void voxelFromBytes(const char* b, VoxelSBR& v)
    {
        std::memcpy(&v.sdf, b, 8); std::memcpy(&v.weight, b + 8, 4); std::memcpy(v.color.data(), b + 12, 3); std::memcpy(&v.albedo, b + 16, 8); std::memcpy(&v.sdf_refined, b + 24, 8);
    }
    float voxel_size_ = 0.004f, truncation_ = 0.02f;
    float integration_weight_sample_ = 10.0f, max_load_factor_ = 0.6f;     // .tsdf header fields kept for a byte-faithful load -> save round trip
    std::vector<value_type> nodes_;
    std::unordered_map<Vec3i, size_t> index_;
};
static_assert(sizeof(Voxel) == 12 && sizeof(VoxelSBR) == 32, "voxel structs must keep the reference's layout (the .tsdf format is a raw dump)");
} // namespace nv
