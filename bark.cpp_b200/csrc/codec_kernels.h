// Host-callable launchers of the EnCodec kernels (codec_kernels.cu).
//
// Every launcher takes n items (clips) of independent lengths L[0..n): item b's activation [C][L_b] is the single-clip layout and sits
// at C * (L_0 + ... + L_{b-1}) in the buffer (item-major), so item b of a batch computes exactly what the same clip computes alone.
#pragma once
#include "model.h"

#include <climits>

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
// A window of each item's signal (the streams of codec_stream.cu): item b's input columns [C][L_b] are the global positions org[b] ..
// org[b] + L_b - 1 of its signal, and the launch computes the n_out[b] outputs from global output first[b] on, [Cout][n_out[b]] per item.
// The reflections apply where the global position is outside the signal: below 0 on the left, past the window's last column on the
// right (a window ends where its signal ends, or its outputs read no further).  A launcher without a window runs whole signals:
// org = first = 0 and every output.  Outputs that read outside a window are refused.
struct CodecWindow { long long org[kCodecMaxItems] = {}, first[kCodecMaxItems] = {}; int n_out[kCodecMaxItems] = {}; };
// strided_conv_1d (ops.cpp:59-75) on x [Cin][L_b]: ELU on the input when elu_in, resid added to the output (stride 1 only).
// y is [Cout][conv1d_out_len(L_b, k, stride)]; the launcher picks the kernel from the contraction length and the stride.
int conv1d(const float * x, int Cin, const int * L, int n, const ConvW & cv, bool elu_in, const float * resid, float * y, cudaStream_t s, int stride = 1,
           const CodecWindow * win = nullptr);
int conv1d_out_len(int T, int k, int stride);
// returns the NG of the convtr1d_lane_kernel<NG> it ran.  With a window, output block t reads input frames t - 1 and t: a window from
// first[b] > 0 on starts with frame first[b] - 1.
int convtr1d(const float * x, int Cin, const int * L, int n, const ConvW & cv, int stride, float * y /*[Cout][L_b*stride]*/, cudaStream_t s,
             const CodecWindow * win = nullptr);
// returns kLstmOne or kLstmBatched.  state (may be null, as may its entries): item b's (h, c) [2][C] before its first step, zeros where
// null, and after its last step (not touched for T_b = 0)
int lstm_layer(const float * x, int C, const int * T, int n, const __half * wih_li, const __half * whh_li, int Kp, const float * bih, const float * bhh,
               const float * skip, float * gi_scratch /*[T_b][4C]*/, float * hbuf /*[2][kCodecMaxItems][C]*/, unsigned * counter, float * out,
               cudaStream_t s, float * const * state = nullptr);
// Copies of column blocks between device matrices of `rows` rows, all in one launch: job j copies [rows][cols[j]] from src[j] (row
// stride src_ld[j]) to dst[j] (row stride dst_ld[j]).  The streams' windows and histories move through it.
constexpr int kColumnCopyJobs = 2 * kCodecMaxItems;
struct ColumnCopies { int n = 0; const float * src[kColumnCopyJobs]; float * dst[kColumnCopyJobs]; int src_ld[kColumnCopyJobs], dst_ld[kColumnCopyJobs], cols[kColumnCopyJobs]; };
void copy_columns(const ColumnCopies & c, int rows, cudaStream_t s);
// load-time re-layout of a transposed-conv weight: [Cin][Cout][k] -> rows [Cout][k][Cin]
void convtr_rows(const __half * src, __half * dst, int Cin, int Cout, int k, cudaStream_t s);

// Resampling (DESIGN.md §16): torchaudio.functional.resample's default sinc_interp_hann filter with an exact summation order, after
// upstream EnCodec's channel down-mix.  Both rates lie in [kResampleMinRate, kResampleMaxRate].
constexpr int kResampleMinRate = 4000, kResampleMaxRate = 384000, kResampleMaxChannels = 8;
// o = sr / g, q = new_sr / g (g = gcd) and the filter's half width w in input frames (0 for equal rates)
void resample_rates(int sr, int new_sr, int * o, int * q, int * w);
// L = ceil(q n / o): samples of n frames at sr resampled to new_sr
long long resample_len(long long n, int sr, int new_sr);
// R(n) = q max(0, floor((n - w) / o)), n for equal rates: the outputs that no frame after the first n can change (DESIGN.md §20)
long long resample_ready(long long n, int sr, int new_sr);
// The taps of sr -> new_sr in double by the rule, rounded to f32, each phase trimmed to its nonzero span; fills t's sizes and returns
// the bytes to upload (phases, then taps; empty for the identity)
std::vector<unsigned char> resample_table(int sr, int new_sr, ResampleTable * t);
// points t at its uploaded bytes
void resample_bind(ResampleTable & t, const void * dev);
// x: n interleaved frames [n][C] (device) -> y [L] (device), L = resample_len(n, t.sr, t.new_sr)
void resample(const float * x, long long n, int C, const ResampleTable & t, float * y, int L, cudaStream_t s);
// A window of one signal (the streams of codec_stream.cu): x holds len interleaved frames [len][C], the global frames org .. org + len
// - 1, and y gets the n_out global outputs from first on.  Global frames below 0, and at or past end (LLONG_MAX while the end is not
// known), read as zeros.  A window whose outputs read, over the filter's full support, a frame it neither holds nor treats as outside
// the signal is refused.
struct ResampleWindow {
    ResampleTable t;
    const float * x = nullptr; float * y = nullptr;
    long long org = 0, first = 0, end = LLONG_MAX;
    int len = 0, n_out = 0, C = 1;
};
// n <= kCodecMaxItems windows of their own tables and formats in one launch (shared memory: the largest item's)
void resample_windows(const ResampleWindow * w, int n, cudaStream_t s);

}  // namespace bark
