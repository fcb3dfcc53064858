// Bitonic sort of 64-bit keys (ascending) on the device, shared by the detection candidates (detect.cu) and the VOC
// AP records (voc_eval.cu).  The kernels live in detect.cu; this header declares their launch sequence.
#pragma once
#include "common.cuh"

namespace effdet {

// Sorts `n` keys as independent segments of `seg` keys each (seg a power of two, n a multiple of seg): a chunk sort of
// up to 2048 keys per CTA in shared memory, then global compare-exchange steps and chunk merges for the larger stages.
// No allocation, no synchronisation; the launch count depends on n and seg only.
int bitonic_sort_launch(uint64_t* keys, int n, int seg, cudaStream_t st);

}  // namespace effdet
