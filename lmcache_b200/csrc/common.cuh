// common.cuh -- error plumbing and small device helpers shared by the libb200kv translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <string>

#include "../../include/b200kv.h"

namespace b200kv {

void set_error(const std::string& msg);   // thread-local last error (api.cu)

#define B2_CHECK_CUDA(expr)                                                                      \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess) {                                                                 \
            ::b200kv::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));             \
            return -1;                                                                           \
        }                                                                                        \
    } while (0)

#define B2_REQUIRE(cond, msg)                                                                    \
    do {                                                                                         \
        if (!(cond)) {                                                                           \
            ::b200kv::set_error(std::string("invalid argument: ") + (msg));                      \
            return -2;                                                                           \
        }                                                                                        \
    } while (0)

// Kernel-parameter copy of the per-plane base pointers and quantiser constants
// (plane nl = kv * L + l).  Lives in the constant bank; indexed dynamically.  3 KB at 256 planes: every parameter block
// that holds one stays under the classic 4 KB kernel-parameter limit (static_asserts next to each).
template <int N>
struct PlaneTableT {
    const uint16_t* p[N];
    float maxq[N];                       // bins // 2 - 1
};
using PlaneTable = PlaneTableT<B200KV_MAX_PLANES>;
constexpr size_t kMaxParamBytes = 4096;

// Planes per layer of a kv_desc (1 for a latent KV, B200KV_KV_LATENT) and its element dtype without the flag.
inline int kv_ppl(const b200kv_kv_desc* kv) { return (kv->dtype & B200KV_KV_LATENT) ? 1 : 2; }
inline int kv_dtype(const b200kv_kv_desc* kv) { return kv->dtype & ~B200KV_KV_LATENT; }

// Fill a PlaneTable from a kv_desc + bins (planes kv * L + l; a latent KV's plane l takes key_bins[l]); returns 0 or <0
// with error set.
int make_plane_table(const b200kv_kv_desc* kv, const float* key_bins, const float* value_bins, PlaneTable* out);

// Row of a token inside its plane.  PAGED: the caller's slot mapping (vLLM's paged KV cache: row = block * block_size
// + offset); every lane of a warp asks for the same token, so the lookup is one broadcast load that hits L1.
template <bool PAGED>
__device__ __forceinline__ int64_t tok_row(const int64_t* slot_map, int64_t tok) {
    if constexpr (PAGED) return __ldg(slot_map + tok);
    else return tok;
}

}  // namespace b200kv
