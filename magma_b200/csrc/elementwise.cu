// magma_b200 — HBM-bound kernels of the hot path (normalisation, rotary, softmax, cross-entropy, gathers,
// label building, reductions, token sampling). All use 128-bit loads/stores where the layout allows, fp32 math, bf16
// storage. The kernels and their C ABI live in fragments that oracle/kernel_host_exec.cpp also compiles.
#include <curand_kernel.h>

#include "common.cuh"

namespace mb200 {

#include "elt_helpers.cuh"
#include "elt_kernels.cuh"
#include "train_kernels.cuh"

namespace {
#include "samp_kernels.cuh"
}  // namespace

// Kernels meant to be resident BESIDE a persistent GEMM CTA (optimizer on its side stream, peer-memory gradient exchange)
// ask for the same shared-memory / L1 split as the GEMM (maximum shared memory): an SM's carve-out is only reconfigured
// when the SM is empty, so a resident block of a kernel that prefers a large L1 keeps a 209 KB GEMM CTA off that SM until
// it leaves — co-residency then degenerates into time slicing. These kernels stream and have no use for L1.
template <typename K>
static void prefer_max_smem_carveout(K kernel) {
  cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}
static void co_resident_kernels_init() {
  static bool done = false;
  if (done) return;
  done = true;
  prefer_max_smem_carveout(adamw_kernel);
  prefer_max_smem_carveout(sumsq_kernel);
  prefer_max_smem_carveout(peer_reduce_bcast_kernel);
  prefer_max_smem_carveout(cast_f32_bf16_kernel);
}

}  // namespace mb200

#include "elt_abi.cuh"
