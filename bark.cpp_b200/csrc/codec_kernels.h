// Host-callable launchers of the EnCodec kernels (codec_kernels.cu).
//
// Every launcher takes n items (clips) of independent lengths L[0..n): item b's activation [C][L_b] is the single-clip layout and sits
// at C * (L_0 + ... + L_{b-1}) in the buffer (item-major), so item b of a batch computes exactly what the same clip computes alone.
#pragma once
#include "model.h"

namespace bark {

// Items of one launch: bounded by the LSTM recurrence, whose CTAs hold h_{t-1} of every item in shared memory ([B][512] floats, 64 KB
// at 32 items) and whose c state takes one thread per (unit, item) (4 units x 32 items of its 512 threads).
constexpr int kCodecMaxItems = 32;

void rvq_decode(const CodecModel & cm, const int32_t * d_codes /*[n_q][T_b] per item*/, int n_q, const int * T, int n, float * x /*[hidden][T_b]*/,
                cudaStream_t s);
// e_j = sum of squares of codeword j (the RVQ encode's codebook norms), embed [n_bins][Hd] -> out [n_bins]
void rvq_norms(const float * embed, int n_bins, int Hd, float * out, cudaStream_t s);
// codes [n_q][T_b] of latent [Hd][T_b] per item through codebooks embed[q] [n_bins][Hd] with their norms; false for shapes outside
// n_q <= 32, n_bins <= 1024, Hd % 32 == 0 and Hd <= 128
bool rvq_encode(const float * const * embed, const float * const * norms, int n_q, int n_bins, int Hd, const float * latent, const int * T, int n,
                int32_t * codes, cudaStream_t s);
// The kernel a convolution launcher ran: conv1d_short_kernel, conv1d_lane_kernel<KW, NG> as kConvLane + 10 KW + NG, conv1d_stream_kernel<KW,
// STRIDE> as kConvStream + 100 KW + STRIDE; the LSTM recurrence of one item or of several.  The pipeline ignores them; the tests count them.
constexpr int kConvShort = 1, kConvLane = 1000, kConvStream = 10000, kLstmOne = 1, kLstmBatched = 2;
// strided_conv_1d (ops.cpp:59-75) on x [Cin][L_b]: ELU on the input when elu_in, resid added to the output (stride 1 only).
// y is [Cout][conv1d_out_len(L_b, k, stride)]; the launcher picks the kernel from the contraction length and the stride.
int conv1d(const float * x, int Cin, const int * L, int n, const ConvW & cv, bool elu_in, const float * resid, float * y, cudaStream_t s, int stride = 1);
int conv1d_out_len(int T, int k, int stride);
// returns the NG of the convtr1d_lane_kernel<NG> it ran
int convtr1d(const float * x, int Cin, const int * L, int n, const ConvW & cv, int stride, float * y /*[Cout][L_b*stride]*/, cudaStream_t s);
// returns kLstmOne or kLstmBatched
int lstm_layer(const float * x, int C, const int * T, int n, const __half * wih_li, const __half * whh_li, int Kp, const float * bih, const float * bhh,
               const float * skip, float * gi_scratch /*[T_b][4C]*/, float * hbuf /*[2][kCodecMaxItems][C]*/, unsigned * counter, float * out,
               cudaStream_t s);
// load-time re-layout of a transposed-conv weight: [Cin][Cout][k] -> rows [Cout][k][Cin]
void convtr_rows(const __half * src, __half * dst, int Cin, int Cout, int k, cudaStream_t s);

// Resampling (DESIGN.md §16): torchaudio.functional.resample's default sinc_interp_hann filter with an exact summation order, after
// upstream EnCodec's channel down-mix.  Both rates lie in [kResampleMinRate, kResampleMaxRate].
constexpr int kResampleMinRate = 4000, kResampleMaxRate = 384000, kResampleMaxChannels = 8;
// L = ceil(q n / o): samples of n frames at sr resampled to new_sr
long long resample_len(long long n, int sr, int new_sr);
// The taps of sr -> new_sr in double by the rule, rounded to f32, each phase trimmed to its nonzero span; fills t's sizes and returns
// the bytes to upload (phases, then taps; empty for the identity)
std::vector<unsigned char> resample_table(int sr, int new_sr, ResampleTable * t);
// points t at its uploaded bytes
void resample_bind(ResampleTable & t, const void * dev);
// x: n interleaved frames [n][C] (device) -> y [L] (device), L = resample_len(n, t.sr, t.new_sr)
void resample(const float * x, long long n, int C, const ResampleTable & t, float * y, int L, cudaStream_t s);

}  // namespace bark
