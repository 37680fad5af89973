// jf_bloom.cuh -- the kernels of sharded Bloom counting: the owner-side --bf-size prefilter in front of the key exchange's
// insertion (insert_keys_bf_kernel, stage_keys_bf_kernel of jf_kernels.cuh) and the fold of two Bloom counters
// (bloom_fold_kernel, jf_bloom.cu).
//
// Like the kernels of four-word keys (jf_wide.cuh) they are instantiated in a translation unit of their own, jf_bloom.cu, and
// jf_engine.cu launches them through the pointers below (typed there, jf_engine.cu: bloom_kernels): split compilation
// assigns functions to partitions over the whole module, and new instantiations next to the engine's kernels would change
// their code.
#ifndef JF_BLOOM_CUH
#define JF_BLOOM_CUH
#include <stddef.h>

namespace jfbl {

struct Kernels {                   // host stubs of the kernels (the argument types are those of namespace jfk)
  const void* insert_keys[5];      // insert_keys_bf_kernel<KW, SB>: (1, 32), (1, 64), (1, 128), (2, 64), (2, 128)
  const void* stage_keys[2];       // stage_keys_bf_kernel<KW>: KW = 1, 2
  const void* fold;                // bloom_fold_kernel
};
const Kernels& kernels();

}  // namespace jfbl
#endif
