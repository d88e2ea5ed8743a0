// capi_common.h -- shared by the extern "C" translation units: the opaque handle, argument-check macros, the row-map helpers and
// the conversions of the key structs of the public header.
#pragma once
#include <cstdint>
#include "../../include/lattigo_b200.h"
#include "composite.h"
#include "engine.h"
#include <nvtx3/nvToolsExt.h>

namespace lgpu {
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
    NvtxRange(const NvtxRange&) = delete;
    NvtxRange& operator=(const NvtxRange&) = delete;
};
}  // namespace lgpu

struct lgpu_ctx {
    lgpu::Ctx c;
};

#define REQUIRE(cond, msg)                 \
    do {                                   \
        if (!(cond)) {                     \
            lgpu::set_error(msg);          \
            return -1;                     \
        }                                  \
    } while (0)
// every device entry point opens an NVTX range named after itself (visible in nsys / ncu --nvtx; a no-op without a tool attached), so that a
// trace of the Go application shows which ring / evaluator method each group of kernels belongs to
#define REQUIRE_DEVICE(ctx) REQUIRE_DEVICE_AS(ctx, __func__)
// the same in a helper that runs on behalf of the entry point `name`
#define REQUIRE_DEVICE_AS(ctx, name)                                                                                             \
    REQUIRE((ctx) && (ctx)->c.device >= 0, "this context was created host-only (device < 0): no device execution");             \
    lgpu::NvtxRange lgpu_nvtx_range_(name)
// the key-switch family moves 128 bits per access: polynomial blocks must be 16-byte aligned with even strides
#define AL(p) ((reinterpret_cast<uintptr_t>(p) & 15u) == 0)
#define REQUIRE_ALIGNED(cond) REQUIRE(cond, "polynomial buffers and evaluation keys must be 16-byte aligned with even strides (words)")

namespace lgpu {
// rows 0..level of ring Q or P -> global limb indices (capi.cu)
int make_rowmap(const Ctx& c, int ring, int level, RowMap& rm);
int make_rowmap_single(const Ctx& c, int ring, int limb, RowMap& rm);
// lgpu_gadget_ct -> GadgetCt: null key or data (null_msg), 16-byte alignment of the data, n_pw2_max <= 0 read as 1 (capi.cu)
int to_gadget_ct(const lgpu_gadget_ct* e, GadgetCt& g, const char* null_msg = "null evaluation key");
// lgpu_galois_keys -> GaloisKeySet: null set, null arrays for n_keys > 0, then every key through to_gadget_ct (capi.cu)
int to_galois_keys(const lgpu_galois_keys* gks, GaloisKeySet& ks);
// [a, a + abytes) and [b, b + bbytes) intersect
bool overlaps(const void* a, size_t abytes, const void* b, size_t bbytes);
}  // namespace lgpu
