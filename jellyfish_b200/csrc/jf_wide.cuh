// jf_wide.cuh -- the kernels of four-word keys (k = 65..128, the wide slot form SB_WIDE of jf_device.cuh).
//
// They are instantiated in their own translation unit, jf_wide.cu, and jf_engine.cu launches them through the pointers
// below (typed there, jf_engine.cu: wide_kernels).  The engine's own module thus holds exactly the kernels of one- and
// two-word keys and compiles them as before the wide form existed: split compilation assigns functions to partitions
// over the whole module, and new instantiations next to them would change their code.
#ifndef JF_WIDE_CUH
#define JF_WIDE_CUH
#include <stddef.h>

namespace jfw {

struct Kernels {                   // host stubs of the kernels (the argument types are those of namespace jfk)
  const void* extract_count;       // extract_kernel<4, SB_WIDE, 0, 512, false>: direct insertion
  const void* extract_query;       // extract_kernel<4, 64, 3, 512, false>: k-mers of a query in input order
  const void* insert_keys;         // insert_keys_kernel<4, SB_WIDE>
  const void* collect;             // collect_kernel<4, SB_WIDE>
  const void* dump_count;          // dump_count_kernel<SB_WIDE>
  const void* dump_emit;           // dump_emit_kernel<4, SB_WIDE>
  const void* lookup;              // lookup_kernel<4, SB_WIDE>
  const void* query_lookup;        // query_lookup_kernel<4, SB_WIDE>
  const void* query_decode;        // query_decode_kernel<4>
  const void* query_format;        // query_format_kernel<4>
  const void* histogram;           // histogram_kernel<SB_WIDE>
  const void* extract_route;       // extract_kernel<4, SB_WIDE, 1, 512, false>: keys bucketed by owning shard
};
const Kernels& kernels();
size_t extract_smem(size_t lut_bytes);    // dynamic shared memory of extract_kernel<4, ...> besides the hash tables

}  // namespace jfw
#endif
