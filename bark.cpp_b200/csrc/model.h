// Device-resident model description: what the loader produces and the kernels consume.
// Mirrors the reference's gpt_hparams / gpt_layer / gpt_model (bark.cpp:49-121) and encodec_model
// (encodec.cpp/encodec.cpp:47-99), but every pointer is HBM and every matrix is in the
// lane-interleaved layout of common.cuh.
#pragma once
#include "common.cuh"

#include <string>
#include <vector>

namespace bark {

struct DMat {                 // 2-D weight [n_out][K] in LI layout (f32 / f16) or q4_0 blocks
    void * p = nullptr;
    int n_out = 0, K = 0, Kp = 0;   // Kp = padded row length in elements
    void * scales = nullptr;        // quantised: f16 block scales [n_out][K/32]; p then holds the 16-byte nibble words (32 B for q8_0) [n_out][K/32]
    void * mins = nullptr, * qh = nullptr;   // experimental types: f16 block minima (q4_1, q5_1), fifth bits (q5_0, q5_1)
    void * p_gm = nullptr; int o_pad = 0;   // second copy in the group-major layout (common.cuh) for the tiled GEMM; rows padded to o_pad
    void * p_rm = nullptr;                  // fast mode only: the row-major [n_out][K] f16 matrix = K-major wgmma operand (fast_kernels.cu); an f16 file's own upload, else its fast_convert copy
    WType type = W_F16;
};

struct GPTLayer {
    float * ln_1_g = nullptr, * ln_1_b = nullptr, * ln_2_g = nullptr, * ln_2_b = nullptr;
    DMat c_attn, c_proj, fc, proj;
};

struct GPTModel {
    // header order of the file (bark.cpp:700-709)
    int32_t n_layer = 0, n_head = 0, n_embd = 0, block_size = 0, bias = 0, n_in_vocab = 0, n_out_vocab = 0,
            n_lm_heads = 0, n_wtes = 0, ftype = 0;
    WType wtype = W_F16;
    void * wte[8] = {nullptr};        // token tables, ORIGINAL row-major layout (gather only)
    float * wpe = nullptr;            // [block_size][E] f32
    float * ln_f_g = nullptr, * ln_f_b = nullptr;
    DMat lm_head[8];
    std::vector<GPTLayer> layers;
    float * mem_k = nullptr, * mem_v = nullptr;   // [L][block_size][E] f32 (bark.cpp:980-981); null for the fine model
    // persistent decode step (decode_kernels.cu): phase table + cross-CTA exchange buffers, built once at load
    bool decode_ok = false;           // the model fits the persistent kernel's fixed capacities (build_decode_tables); otherwise per-op stepping
    void * d_phases = nullptr, * d_layer_vecs = nullptr;
    unsigned long long * gx = nullptr, * gq = nullptr, * gk = nullptr, * gv = nullptr, * gatt = nullptr, * gff = nullptr, * gscores = nullptr;
    float * glogits = nullptr;
    // per-model statistics, same meaning as gpt_model::t_* (bark.cpp:114-118)
    int64_t t_sample_us = 0, t_predict_us = 0, t_main_us = 0, n_sample = 0;
};

struct ConvW { __half * w = nullptr; float * b = nullptr; int k = 0, cin = 0, cout = 0, Kp = 0; };   // w: LI16 rows (conv: [Cout] x Cin*k; transposed conv: [Cout*k] x Cin)

constexpr int kMaxCodebooks = 32;          // codebooks of the 24 kHz EnCodec (24 kbps)

// The 24 kHz EnCodec's time axis: the decoder up-samples by the ratios in this order and the encoder down-samples by them in reverse,
// so a latent frame is kCodecHop samples.  The final k=7 convolutions reflect-pad 6 frames: a clip needs kCodecMinFrames frames, that
// is kCodecMinSamples samples (the reference reads out of bounds below that).
constexpr int kCodecRatios[4] = {8, 5, 4, 2};
constexpr int kCodecHop = kCodecRatios[0] * kCodecRatios[1] * kCodecRatios[2] * kCodecRatios[3];   // 320
constexpr int kCodecMinFrames = 7;
constexpr int kCodecMinSamples = kCodecHop * (kCodecMinFrames - 1) + 1;                               // 1921

struct CodecLSTM {                          // two layers (encodec.cpp/lstm.h); the second's input is added to its output
    __half * ih_w[2] = {nullptr, nullptr}, * hh_w[2] = {nullptr, nullptr};   // [4H] x H, LI16 rows of Kp
    int Kp = 0;
    float  * ih_b[2] = {nullptr, nullptr}, * hh_b[2] = {nullptr, nullptr};
};

struct CodecModel {
    int hidden_dim = 128, n_filters = 32, kernel_size = 7, res_kernel = 3, n_bins = 1024;
    ConvW init, final_conv;
    CodecLSTM lstm;
    struct Block { ConvW us, c1, c2, sc; } blk[4];   // us: transposed conv
    int bandwidth = 24, sample_rate = 24000;           // the file's hyper-parameters (kbps, Hz)
    int n_q = 0;                            // codebooks loaded: 0..n_q-1
    float * embed[kMaxCodebooks] = {nullptr};        // codebooks, [n_bins][hidden] f32
    float * embed_norm[kMaxCodebooks] = {nullptr};   // their rows' sums of squares [n_bins] (RVQ encode)
    struct Encoder {                        // encoder.* tensors (encodec.cpp/encoder.h:8-37); a file may lack them all
        bool present = false;
        ConvW init, final_conv;
        struct Block { ConvW sc, c1, c2, ds; } blk[4];   // ds: down-sampling conv, k = 2r, stride r
        CodecLSTM lstm;
    } enc;
};

// Device buffers owned by one context, freed together by release()
struct DeviceArena {
    std::vector<void *> allocs;
    void * alloc(size_t bytes);             // cudaMalloc'ed and recorded (loader.cu)
    void release();
};

// The taps of one rate pair sr -> new_sr (DESIGN.md §16), built on the host by resample_table and bound to device memory by
// resample_bind (codec_kernels.cu).  o = sr / g, q = new_sr / g (g = gcd), w the filter's half width in input samples; phase j has
// phase[j] = {first m, count, offset into taps, 0}.  sr == new_sr is the identity (the down-mix alone) and has no taps.  Outputs go
// tile per CTA with smem floats of shared memory: the tile's input window.
struct ResampleTable {
    int sr = 0, new_sr = 0, o = 1, q = 1, w = 0, tile = 0, smem = 0;
    const int4 * phase = nullptr;
    const float * taps = nullptr;
};

// EnCodec scratch for one launch's items (T frames in all), grown on demand by codec_scratch (codec_pipeline.cu), freed by release()
struct CodecScratch {
    float * buf[3] = {nullptr, nullptr, nullptr}; size_t cap = 0;   // ping-pong activations (floats), item-major
    float * gi = nullptr;                                            // LSTM input projections
    float * hbuf = nullptr; unsigned * counter = nullptr;            // LSTM hidden-state exchange [2][items][512] + grid barrier counter
    int32_t * codes = nullptr; size_t codes_cap = 0;                 // [n_q][T_b] per item
    float * stage = nullptr; size_t stage_cap = 0;                   // one resampled item's interleaved source frames (floats)
    std::vector<std::pair<ResampleTable, void *>> tables;            // resampling taps per rate pair, with their device allocation
    void release();
};

// Scratch activations for one GPT evaluation of up to `max_rows` positions.
struct Workspace {
    int max_rows = 0, E = 0;
    float * x = nullptr;        // residual stream [rows][E]
    void  * act = nullptr;      // LI-layout activation operand for the next matmul [rows][max(Kp)]
    void  * act2 = nullptr;     // second operand buffer (GELU output feeding mlp/c_proj)
    float * q = nullptr;        // [rows][E]
    float * kbuf = nullptr, * vbuf = nullptr;   // fine model K/V [rows][E]
    float * scores = nullptr;   // [B <= 8][H][max_kv] (attention_batch) or [H][N][n_kv] for N <= attn_tiled_max_rows (attention)
    float * logits = nullptr;   // [rows][n_out]
    int32_t * tok = nullptr;    // device copy of the ids fed this step
};

}  // namespace bark
