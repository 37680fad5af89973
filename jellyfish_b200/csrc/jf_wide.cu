// jf_wide.cu -- instantiations of the kernels of four-word keys (jf_wide.cuh).
// The kernel headers are compiled here under a namespace of their own: their non-template kernels (scans, zeroing) are
// defined by jf_engine.cu as well, and the argument structures are laid out identically in both.
#include <cuda_runtime.h>
#define jfk jfk_wide
#include "jf_extract.cuh"
#include "jf_dump.cuh"
#include "jf_query.cuh"
#undef jfk
#include "jf_wide.cuh"

namespace jfw {
using namespace jfk_wide;

const Kernels& kernels() {
  static const Kernels k = {
    (const void*)extract_kernel<4, SB_WIDE, 0, 512, false>,
    (const void*)extract_kernel<4, 64, 3, 512, false>,
    (const void*)insert_keys_kernel<4, SB_WIDE>,
    (const void*)collect_kernel<4, SB_WIDE>,
    (const void*)dump_count_kernel<SB_WIDE>,
    (const void*)dump_emit_kernel<4, SB_WIDE>,
    (const void*)lookup_kernel<4, SB_WIDE>,
    (const void*)query_lookup_kernel<4, SB_WIDE>,
    (const void*)query_decode_kernel<4>,
    (const void*)query_format_kernel<4>,
    (const void*)histogram_kernel<SB_WIDE>,
    (const void*)extract_kernel<4, SB_WIDE, 1, 512, false>,
  };
  return k;
}

size_t extract_smem(size_t lut_bytes) { return ((sizeof(ExtractSmemT<512, PRE_WIDE>) + 15) & ~(size_t)15) + lut_bytes; }

}  // namespace jfw
