// Host build of nerf_rpn_b200/csrc/anchor_mask.cuh (TEST ONLY): the padding-mask functions of nrpn_anchor_padding_mask compiled as
// plain C++ to check them against the reference's get_padding_masks on GPU-less boxes.  The loops below stand in for the entry point
// and the thread grid of targets.cu; the product never uses this file.
#include <cstdint>
#define __device__
#define __host__
#include "../../nerf_rpn_b200/csrc/anchor_mask.cuh"

using namespace nrpn;

// ori: n x 3, grid_dims: n_levels x 3; out: n x total bytes.  Returns total.
extern "C" long long shim_anchor_padding_mask(const int* ori, int n, int px, int py, int pz, const int* grid_dims, int n_levels, int num_anchors,
                                              uint8_t* out) {
    const int pad[3] = {px, py, pz};
    AnchorMaskLevel lv[kMaskMaxLevels];
    long long begin = 0;
    for (int l = 0; l < n_levels; ++l) {
        lv[l].begin = begin;
        for (int a = 0; a < 3; ++a) lv[l].grid[a] = grid_dims[3 * l + a];
        begin += (long long)num_anchors * lv[l].grid[0] * lv[l].grid[1] * lv[l].grid[2];
    }
    const long long total = begin;
    if (!out) return total;
    int lim[kMaskMaxLevels][3];
    for (int i = 0; i < n; ++i) {
        for (int l = 0; l < n_levels; ++l)
            for (int a = 0; a < 3; ++a) lim[l][a] = anchor_mask_limit(ori[3 * i + a], pad[a], lv[l].grid[a]);
        for (long long k = 0; k < total; ++k) out[(long long)i * total + k] = anchor_mask_value(lv, lim, n_levels, num_anchors, k);
    }
    return total;
}
