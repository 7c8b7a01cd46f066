// Row-sharded fine pass over the GPUs of one NVLink domain (BASELINE.json configs[4]; SURVEY.md §8e).
//
// The six passes of a 1024-frame window are a dependency chain (pass nn embeds the codebooks passes 2..nn-1 produced,
// bark.cpp:1457-1463, 2015-2039), so codebooks do not shard.  ROWS do: LayerNorm, the mat-muls, GELU and the lm_head are row-local,
// and the non-causal attention (bark.cpp:1495-1530) needs every row's K and V but only its own Q.  Rank r of W evaluates rows
// [r * 1024 / W, (r + 1) * 1024 / W):
//   * the QKV mat-mul's epilogue stores each K / V row into the local buffer AND into the W - 1 peers' buffers over NVLink
//     (peer pointers from CUDA IPC): the per-layer all-gather is fused into the kernel that produces the data;
//   * one flag-based cross-GPU barrier per layer (st.release.sys / ld.acquire.sys on peer memory) orders those stores before the
//     attention reads; K / V are double-buffered by layer parity, so one barrier per layer is enough;
//   * sampling keeps the reference's RNG order: the host draws the window's 1024 uniforms per pass in order and rank r consumes
//     its slice (draw index of (pass, row) is closed-form); the 1024 / W sampled ids are published to every peer the same way.
// Every rank ends up with the same fine tokens, bit-identical to the single-GPU run: each row's arithmetic is exactly what the
// unsharded kernels do for that row.  No NCCL on the data path; process-per-GPU (torchrun) hands the IPC handles around.
#include "../../include/bark_b200.h"
#include "context.h"
#include "gpt_kernels.h"

namespace bark {

namespace {

struct PeerFlags { unsigned * flags[8]; };

// Cross-GPU barrier: thread t tells peer t that this rank has arrived at `epoch`, then waits until peer t has told us the same.
// Runs after the producing kernel in stream order, so the release store publishes that kernel's peer stores as well.
__global__ void xgpu_barrier_kernel(PeerFlags P, int rank, int world, unsigned epoch, unsigned * err) {
    const int t = threadIdx.x;
    if (t >= world) return;
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(P.flags[t] + rank), "r"(epoch) : "memory");
    const unsigned * mine = P.flags[rank] + t;
    const long long t0 = clock64();
    for (;;) {
        unsigned v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
        if ((int)(v - epoch) >= 0) break;
        if (clock64() - t0 > 8000000000ll) { *err = 1u; break; }       // a peer that never arrives must not hang this GPU
        __nanosleep(100);
    }
}

struct PeerIds { int32_t * ids[8]; };
__global__ void publish_ids_kernel(PeerIds P, int world, const int32_t * __restrict__ local, int row0, int rows) {
    const int p = blockIdx.x;
    for (int i = threadIdx.x; i < rows; i += blockDim.x) P.ids[p][row0 + i] = local[i];
}

}  // namespace

// layout of the one IPC-exported allocation per rank
static size_t shard_kv_floats(const GPTModel & m) { return (size_t) 1024 * m.n_embd; }
static size_t shard_bytes(const GPTModel & m) { return 4 * shard_kv_floats(m) * 4 + 1024 * 4 + 256; }       // K0 V0 K1 V1 | ids[1024] | flags[64]
static float * shard_k(unsigned char * base, const GPTModel & m, int parity) { return (float *) base + (size_t)(2 * parity) * shard_kv_floats(m); }
static float * shard_v(unsigned char * base, const GPTModel & m, int parity) { return (float *) base + (size_t)(2 * parity + 1) * shard_kv_floats(m); }
static int32_t * shard_ids(unsigned char * base, const GPTModel & m) { return (int32_t *)(base + 4 * shard_kv_floats(m) * 4); }
static unsigned * shard_flags(unsigned char * base, const GPTModel & m) { return (unsigned *)(base + 4 * shard_kv_floats(m) * 4 + 1024 * 4); }

static bool shard_barrier(bark_context * ctx) {
    ShardState & S = ctx->shard;
    PeerFlags P{};
    for (int p = 0; p < S.world; p++) P.flags[p] = shard_flags(S.peer[p], ctx->fine);
    S.epoch++;
    BARK_LAUNCH(xgpu_barrier_kernel, 1, 32, 0, ctx->stream, P, S.rank, S.world, S.epoch, S.d_err);
    return true;
}

// This rank's rows [row0, row0 + rows) store layer il's K / V rows into the local buffer and every peer's (buffer pair il & 1); the
// barrier after the QKV mat-mul orders those stores before any rank's attention reads all 1024 rows.
void ShardKV::store(bark_context * ctx, const GPTModel & m, int il, int rows, MatmulEpilogue & qkv) const {
    ShardState & S = ctx->shard;
    const size_t at = (size_t) row0 * m.n_embd;
    qkv.k_out = shard_k(S.local, m, il & 1) + at; qkv.v_out = shard_v(S.local, m, il & 1) + at;
    for (int p = 0; p < S.world; p++) if (p != S.rank) {
        qkv.k_peer[qkv.n_peer] = shard_k(S.peer[p], m, il & 1) + at; qkv.v_peer[qkv.n_peer] = shard_v(S.peer[p], m, il & 1) + at; qkv.n_peer++;
    }
    S.nvlink_bytes += (unsigned long long) qkv.n_peer * 2ull * rows * m.n_embd * 4ull;         // the fused all-gather
}

void ShardKV::attend(bark_context * ctx, const GPTModel & m, int il, int rows, const ActLayout & a) const {
    ShardState & S = ctx->shard;
    Workspace & ws = ctx->ws;
    shard_barrier(ctx);
    attention(ws.q, shard_k(S.local, m, il & 1), shard_v(S.local, m, il & 1), rows, 1024, 0, m.n_embd, m.n_head, false, ws.scores, ws.act, a.wt, a.kpE, ctx->stream);
}

// One pass over this rank's rows; logits of those rows are left in ws.logits [rows][n_out].
bool fine_eval_shard(bark_context * ctx, const int32_t * in_buffer, int nn) {
    GPTModel & m = ctx->fine;
    const int rows = 1024 / ctx->shard.world, row0 = ctx->shard.rank * rows;
    if (is_quant(m.wtype)) { fprintf(stderr, "%s: the row-sharded fine pass runs f32 / f16 weights\n", __func__); return false; }
    const int64_t t0 = now_us();
    if (!fine_embed(ctx, in_buffer, nn, row0, rows, __func__)) return false;
    run_layers(ctx, m, rows, ShardKV{row0});
    output_head(ctx, m, ctx->ws.x, rows, m.lm_head[nn - 1], ctx->ws.logits);
    m.t_predict_us += now_us() - t0;
    return true;
}

// Samples this rank's rows with ITS slice of the window's uniforms (the host RNG advances by all 1024 draws, as the reference's
// loop over the rows does), then gathers the 1024 ids of the pass on every rank.
bool sample_shard(bark_context * ctx, std::mt19937 & rng, int n, float temp, int32_t * out_all /*[1024]*/) {
    GPTModel & m = ctx->fine;
    ShardState & S = ctx->shard;
    cudaStream_t s = ctx->stream;
    const int rows = 1024 / S.world, row0 = S.rank * rows;
    const int64_t t0 = now_us();
    if (temp != 0.0f) for (int r = 0; r < 1024; r++) {
        const double u = std::generate_canonical<double, 53>(rng);
        if (r >= row0 && r < row0 + rows) ctx->h_u[r - row0] = u;
    }
    if (sample_and_replay(ctx, ctx->last_logits, m.n_out_vocab, 0, n, rows, temp, false) > 0) {     // the peers must get the replayed ids
        BARK_CUDA_CHECK(cudaMemcpyAsync(ctx->d_stok, ctx->h_stok, (size_t) rows * 4, cudaMemcpyHostToDevice, s)); g_h2d_bytes += (size_t) rows * 4;
    }
    PeerIds P{};
    for (int p = 0; p < S.world; p++) P.ids[p] = shard_ids(S.peer[p], m);
    BARK_LAUNCH(publish_ids_kernel, S.world, 128, 0, s, P, S.world, ctx->d_stok, row0, rows);
    S.nvlink_bytes += (unsigned long long)(S.world - 1) * rows * 4ull;
    shard_barrier(ctx);
    BARK_CUDA_CHECK(cudaMemcpyAsync(ctx->h_tok, shard_ids(S.local, m), 1024 * 4, cudaMemcpyDeviceToHost, s)); g_d2h_bytes += 1024 * 4;
    unsigned err = 0;
    BARK_CUDA_CHECK(cudaMemcpyAsync(&err, S.d_err, 4, cudaMemcpyDeviceToHost, s));
    BARK_CUDA_CHECK(cudaStreamSynchronize(s));
    if (err) { fprintf(stderr, "%s: a peer GPU did not reach the barrier (rank %d of %d)\n", __func__, S.rank, S.world); return false; }
    memcpy(out_all, ctx->h_tok, 1024 * 4);
    m.t_sample_us += now_us() - t0;
    m.n_sample += 1024;                                                       // the pass sampled 1024 rows job-wide, like the reference counts them
    return true;
}

}  // namespace bark

using namespace bark;

// rank / world of this context in a row-sharded fine stage; writes this rank's 64-byte CUDA IPC handle to handle_out
extern "C" int bark_b200_shard_init(struct bark_context * ctx, int rank, int world, void * handle_out) {
    return with_context(ctx, __func__, 0, [&] {
        if (!handle_out || world < 1 || world > 8 || rank < 0 || rank >= world || 1024 % world) return 0;
        ShardState & S = ctx->shard;
        if (S.local) return 0;
        S.rank = rank; S.world = world;
        const size_t bytes = shard_bytes(ctx->fine);
        if (cudaMalloc((void **) &S.local, bytes) != cudaSuccess) { (void) cudaGetLastError(); return 0; }
        BARK_CUDA_CHECK(cudaMemset(S.local, 0, bytes));
        S.d_err = (unsigned *) ctx_alloc(ctx, 16); BARK_CUDA_CHECK(cudaMemset(S.d_err, 0, 16));
        cudaIpcMemHandle_t h;
        if (cudaIpcGetMemHandle(&h, S.local) != cudaSuccess) { fprintf(stderr, "bark_b200_shard_init: cudaIpcGetMemHandle failed: %s\n", cudaGetErrorString(cudaGetLastError())); return 0; }
        static_assert(sizeof(h) == 64, "CUDA IPC handles are 64 bytes");
        memcpy(handle_out, &h, 64);
        S.peer[rank] = S.local;
        return 1;
    });
}

// all_handles: world x 64 bytes, rank order (what every rank's bark_b200_shard_init returned, all-gathered by the caller)
extern "C" int bark_b200_shard_connect(struct bark_context * ctx, const void * all_handles) {
    return with_context(ctx, __func__, 0, [&] {
        if (!all_handles || !ctx->shard.local) return 0;
        ShardState & S = ctx->shard;
        for (int p = 0; p < S.world; p++) {
            if (p == S.rank) continue;
            cudaIpcMemHandle_t h; memcpy(&h, (const unsigned char *) all_handles + (size_t) p * 64, 64);
            void * ptr = nullptr;
            const cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) { fprintf(stderr, "bark_b200_shard_connect: cudaIpcOpenMemHandle for rank %d failed: %s\n", p, cudaGetErrorString(e)); (void) cudaGetLastError(); return 0; }
            S.peer[p] = (unsigned char *) ptr;
        }
        S.on = true;
        return 1;
    });
}

extern "C" unsigned long long bark_b200_shard_nvlink_bytes(struct bark_context * ctx, int reset) {
    return with_context(ctx, __func__, 0ull, [&] {
        const unsigned long long v = ctx->shard.nvlink_bytes;
        if (reset) ctx->shard.nvlink_bytes = 0;
        return v;
    });
}
