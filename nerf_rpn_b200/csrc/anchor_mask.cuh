// Per-anchor padding mask of a padded batch (AnchorGenerator3D.get_padding_masks, anchor.py:124-152, flattened by
// RegionProposalNetwork.get_padding_masks, rpn.py:231-238), as __host__ __device__ functions so that tests/host_shim can run the
// same code on a GPU-less box against the reference.  The kernel around them is in targets.cu.
//   anchor_mask_limit : number of real voxels of one axis of one level, ceil(ori / (padded // grid))
//   anchor_mask_value : 1 / 0 for one flat anchor index (level, voxel (x,y,z) row-major, anchor) of one scene
#pragma once
#include <stdint.h>

namespace nrpn {

constexpr int kMaskMaxLevels = 8;

struct AnchorMaskLevel {
    long long begin;        // first flat anchor index of the level
    int grid[3];            // the level's feature-map extent
};

// The reference computes stride = mesh_size // grid (integer division, so a padded depth of 130 over a P2 grid of 33 gives 3, not 4)
// and limit = ceil(ori_size / stride) in float32; for extents below 2^24 the float quotient rounds to an integer only when it is one,
// so the integer ceiling is the same number.
__host__ __device__ inline int anchor_mask_limit(int ori, int padded, int grid) {
    const int stride = padded / grid;
    return (ori + stride - 1) / stride;
}

// lim: the n_levels x 3 limits of one scene.
__host__ __device__ inline uint8_t anchor_mask_value(const AnchorMaskLevel* lv, const int (*lim)[3], int n_levels, int num_anchors, long long k) {
    int l = 0;
    while (l + 1 < n_levels && k >= lv[l + 1].begin) ++l;
    long long v = (k - lv[l].begin) / num_anchors;
    const int z = (int)(v % lv[l].grid[2]); v /= lv[l].grid[2];
    const int y = (int)(v % lv[l].grid[1]);
    const int x = (int)(v / lv[l].grid[1]);
    return (x < lim[l][0] && y < lim[l][1] && z < lim[l][2]) ? 1 : 0;
}

}  // namespace nrpn
