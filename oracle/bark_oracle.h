/* TEST INFRASTRUCTURE — CPU oracle for the bark.cpp hot path.  NOT product code.
 *
 * A plain-C restatement of the arithmetic the reference executes for
 *   - the causal GPT forward (bark.cpp:1186-1414) and its per-step driver (bark.cpp:1586-1643),
 *   - the non-causal fine GPT forward (bark.cpp:1416-1584, 1907-1959),
 *   - host sampling (bark.cpp:184-270 + libstdc++ bits/random.tcc),
 *   - the three stage loops (bark.cpp:1645-1701, 1745-1863, 1961-2059),
 *   - the EnCodec decoder (encodec.cpp/{quantizer.h:78-111, decoder.h:43-113, lstm.h:22-78, ops.cpp}),
 * with ggml's CPU kernels restated in the AVX2/FMA lane order of the pinned reference build
 * (oracle/Makefile: -mavx2 -mfma -mf16c; SURVEY.md App. C).
 *
 * Pinning: every function here is checked bit-for-bit against the outputs of the unmodified reference
 * (oracle/_ref/libbark_ref.so, compiled by oracle/Makefile) stored in tests/golden/ (tests/test_oracle_vs_ref.py,
 * tests/test_oracle_golden.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load this library.
 */
#ifndef BARK_ORACLE_H
#define BARK_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct orc_ctx orc_ctx;

orc_ctx * orc_load(const char * path, uint32_t seed);
void      orc_free(orc_ctx * c);
void      orc_reseed(orc_ctx * c, uint32_t seed);
/* which: 0 semantic, 1 coarse, 2 fine.  out[10] in file-header order (bark.cpp:700-709) */
void      orc_hparams(orc_ctx * c, int which, int32_t * out);
void      orc_set_params(orc_ctx * c, float temp, float fine_temp, float min_eos_p, int n_steps_text_encoder);

/* tokenizer (bark.cpp:558-662): fills 513 ids */
void orc_tokenize(orc_ctx * c, const char * text, int32_t * out513);

/* one causal-GPT evaluation; mirrors bark_eval_encoder_internal (bark.cpp:1586) */
int  orc_gpt_eval(orc_ctx * c, int which, const int32_t * tokens, int n, int * n_past, int merge_ctx, float * logits_out);
/* one fine pass; in_buffer [8][1024]; logits_out [1024][n_out_vocab] (bark.cpp:1907) */
int  orc_fine_eval(orc_ctx * c, const int32_t * in_buffer, int nn, float * logits_out);
/* gpt_sample (bark.cpp:249) on the context's mt19937 */
int  orc_sample(orc_ctx * c, const float * logits, int n, float temp, float * eos_p);

/* stage loops; return counts.  Buffers sized by the caller (<=768 semantic, frames<=1024) */
int  orc_semantic(orc_ctx * c, const int32_t * prompt513, int32_t * out);
int  orc_coarse(orc_ctx * c, const int32_t * semantic, int n_semantic, int32_t * out_Tx2);
int  orc_fine(orc_ctx * c, const int32_t * coarse_Tx2, int n_frames, int32_t * out_Tx8);
/* EnCodec decode; codes [8][T]; returns samples (320*T) written to out */
int  orc_encodec_decode(orc_ctx * c, const int32_t * codes_8xT, int T, float * out);
/* full bark_generate_audio (bark.cpp:2125); audio_out must hold 320*1024 floats.  Token buffers may be NULL. */
int  orc_generate(orc_ctx * c, const char * text, int32_t * semantic, int * n_semantic,
                  int32_t * coarse, int32_t * fine, int * n_frames, float * audio_out);

/* unit-level entry points used by the op-level tests */
float    orc_vec_dot_f16(int n, const uint16_t * x, const uint16_t * y);
float    orc_vec_dot_f32(int n, const float * x, const float * y);
uint16_t orc_f32_to_f16(float f);
float    orc_f16_to_f32(uint16_t h);
void     orc_gelu_table(uint16_t * out65536);
void     orc_norm(int n, const float * x, float * y, float eps);
void     orc_soft_max(int n, const float * x, float * y);   /* row soft_max as ggml.c:13953 with scale 1 */
float    orc_v_expf(float x);
void     orc_mt_seed(uint32_t * state625, uint32_t seed);
uint32_t orc_mt_next(uint32_t * state625);
/* known-answer hooks: the reference's own op tests (ggml/tests/test-conv1d.cpp, test-conv-transpose-1d.cpp) through the codec's conv cores */
void     orc_test_conv1d(const float * w, int k, int Cin, int Cout, const float * x, int T, int p0, float * y);
void     orc_test_convtr1d(const float * w, int k, int Cout, int Cin, const float * x, int T, int stride, float * y);

#ifdef __cplusplus
}
#endif
#endif
