// Internal (not exported) declarations shared by the two convolution translation units.
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

// Launch with programmatic stream serialization (the kernel must call ptx::pdl_wait() before reading its inputs): the
// prologue of layer i+1 (barrier init, tensor-map prefetch) overlaps the tail of layer i, also inside a captured CUDA graph.
// NRPN_PDL=0 falls back to ordinary stream-ordered launches.  It is applied only to latency-bound launches of at most 2 tiles
// per SM slot (`small`); NRPN_PDL=2 forces it on for every launch.
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

// conv3d_slab.cu: halo-slab kernel for 64 -> (<=64)-channel stride-1 convolutions with a full box of filter taps.
// Returns true when the descriptor is of that shape (the caller then launches it with conv3d_slab_launch).
bool conv3d_slab_eligible(const nrpn_conv_desc* d);
int conv3d_slab_launch(const nrpn_conv_desc* d, cudaStream_t st);

}  // namespace nrpn
