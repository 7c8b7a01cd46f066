// Host-callable launchers of the EnCodec kernels (codec_kernels.cu).
#pragma once
#include "model.h"

namespace bark {

void rvq_decode(const CodecModel & cm, const int32_t * d_codes /*[n_q][T]*/, int n_q, int T, float * x /*[hidden][T]*/, cudaStream_t s);
// e_j = sum of squares of codeword j (the RVQ encode's codebook norms), embed [n_bins][Hd] -> out [n_bins]
void rvq_norms(const float * embed, int n_bins, int Hd, float * out, cudaStream_t s);
// codes [n_q][T] of latent [Hd][T] through codebooks embed[q] [n_bins][Hd] with their norms; false for shapes outside
// n_q <= 32, n_bins <= 1024, Hd % 32 == 0 and Hd <= 128
bool rvq_encode(const float * const * embed, const float * const * norms, int n_q, int n_bins, int Hd, const float * latent, int T, int32_t * codes,
                cudaStream_t s);
// strided_conv_1d (ops.cpp:59-75) on x [Cin][T]: ELU on the input when elu_in, resid added to the output (stride 1 only).
// y is [Cout][conv1d_out_len(T, k, stride)]; the launcher picks the kernel from the contraction length and the stride.
void conv1d(const float * x, int Cin, int T, const ConvW & cv, bool elu_in, const float * resid, float * y, cudaStream_t s, int stride = 1);
int conv1d_out_len(int T, int k, int stride);
void convtr1d(const float * x, int Cin, int T, const ConvW & cv, int stride, float * y /*[Cout][T*stride]*/, cudaStream_t s);
void lstm_layer(const float * x, int C, int T, const __half * wih_li, const __half * whh_li, int Kp, const float * bih, const float * bhh,
                const float * skip, float * gi_scratch /*[T][4C]*/, float * hbuf /*[2][C]*/, unsigned * counter, float * out, cudaStream_t s);
// load-time re-layout of a transposed-conv weight: [Cin][Cout][k] -> rows [Cout][k][Cin]
void convtr_rows(const __half * src, __half * dst, int Cin, int Cout, int k, cudaStream_t s);

}  // namespace bark
