// tensor-core (wgmma) linear layer (linear_tc.cu)
#pragma once
#include "linear_f32.cuh"

namespace dyn {

struct TcLinArgs {
  Seg seg[4];
  int nseg;
  const float* row_scale;
  const void* Wp;   // packed bf16 chunk images (tc_pack_weight)
  const float* b;
  float* Y;
  int ldy;
  long long M;
  int N, K, Npad, nchunks, act;
};

size_t tc_packed_bytes(int N, int K);
int tc_pack_weight(const float* W, int N, int K, void* out, cudaStream_t st);
// same semantics as launch_linear(); W is taken from `packed_w`
int launch_linear_tc(const LinArgs& a, const void* packed_w, cudaStream_t st);

}  // namespace dyn
