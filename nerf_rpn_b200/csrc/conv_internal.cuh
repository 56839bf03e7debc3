// Internal (not exported) declarations shared by the convolution translation units (igemm, halo-slab, weight gradient).
#pragma once
#include <cuda.h>
#include <cstdlib>
#include <utility>
#include "common.cuh"

namespace nrpn {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled through the runtime's driver entry point table (the library does not link libcuda).
inline EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// Encodes a tiled tensor map with the settings every convolution map shares: 128B swizzle, 256B L2 promotion, out-of-bounds
// elements read as zero (no NaN fill), unit element strides.  The bf16 default moves fp16 data just as well: TMA copies bytes.
// NRPN_ERR_NO_DEVICE without the driver entry point; NRPN_ERR_CUDA (and nrpn_last_cuda_error) when the driver refuses the map.
template <int RANK>
inline int encode_tmap(CUtensorMap* map, const void* base, const cuuint64_t (&dims)[RANK], const cuuint64_t (&strides)[RANK - 1],
                       const cuuint32_t (&box)[RANK], CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) {
    EncodeTiledFn encode = get_encode();
    if (!encode) return NRPN_ERR_NO_DEVICE;
    cuuint32_t estr[RANK];
    for (int i = 0; i < RANK; ++i) estr[i] = 1;
    const CUresult r = encode(map, dt, RANK, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { g_last_cuda_error = (int)r; return NRPN_ERR_CUDA; }
    return NRPN_OK;
}

// Launch with programmatic stream serialization (the kernel must call ptx::pdl_wait() before reading its inputs): the
// prologue of layer i+1 (barrier init, tensor-map prefetch) overlaps the tail of layer i, also inside a captured CUDA graph.
// NRPN_PDL=0 falls back to ordinary stream-ordered launches.  It is applied only where the caller passes `small`: every
// implicit-GEMM launch (dynamically scheduled tiles), and latency-bound halo-slab launches of at most 2 tiles per SM; NRPN_PDL=2
// forces it on for every launch.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool small, Args&&... args) {
    static const int mode = [] { const char* e = getenv("NRPN_PDL"); return e ? (e[0] - '0') : 1; }();
    const bool enabled = mode == 2 || (mode == 1 && small);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = enabled ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// The epilogues store an output channel pair as one 4-byte (16-bit y) or 8-byte (fp32 y) word, and load a residual pair as one
// 4-byte word and a shift pair as one 8-byte word.  Row pitches are multiples of 8 elements, so aligned base pointers suffice.
inline bool conv_pairs_aligned(const nrpn_conv_desc* d) {
    if (reinterpret_cast<uintptr_t>(d->shift) % 8 != 0) return false;
    for (int l = 0; l < d->n_levels; ++l) {
        const nrpn_conv_level& S = d->level[l];
        if (reinterpret_cast<uintptr_t>(S.y) % (d->out_fp32 ? 8 : 4) != 0 || reinterpret_cast<uintptr_t>(S.res) % 4 != 0) return false;
    }
    return true;
}

// conv3d_slab.cu: halo-slab kernel for 64 -> (<=64)-channel stride-1 convolutions with a full box of filter taps.
// Returns true when the descriptor is of that shape (the caller then launches it with conv3d_slab_launch, on a descriptor
// nrpn_conv3d_fprop has validated).
bool conv3d_slab_eligible(const nrpn_conv_desc* d);
int conv3d_slab_launch(const nrpn_conv_desc* d, cudaStream_t st);

}  // namespace nrpn
