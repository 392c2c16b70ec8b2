// Host-side interface of the GJK passes (kernels in hfb_gjkpass.cu).
#pragma once
#include <cuda_runtime.h>

#include "hfb_batch.cuh"

// bytes of solver state for n pairs
size_t gjk_pass_state_bytes(size_t n);
// GJK over the class-sorted range [*a.range_lo, *a.range_hi) of a.index_list (at most n pairs) in `npass` passes of
// steps[0], steps[1], ... iterations (the last pass runs to convergence).  Every pass writes the result records, or
// EPA queue items, of the pairs it finished.  gjk_passes_first: the first pass; gjk_passes_rest: the other passes.
// Between the two the caller may start EPA over the queue so far on a side stream.  `counts`: npass words.  Return a
// cudaError_t as int.
int gjk_passes_first(const BatchArgs& a, int mode, unsigned n, void* state, uint32_t* list_a, unsigned* counts,
                     const int* steps, int npass, int num_sms, cudaStream_t s, int* launches);
int gjk_passes_rest(const BatchArgs& a, int mode, unsigned n, void* state, uint32_t* list_a, uint32_t* list_b,
                    unsigned* counts, const int* steps, int npass, int num_sms, cudaStream_t s, int* launches);
