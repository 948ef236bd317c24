// libssb200.so -- sm_90a kernels + C ABI for the SoundSpaces audio observation.
// See include/ssb200.h for the boundary and DESIGN.md for the data layout.
//
// Kernels (all hand written, FP32 SIMT; no cuFFT / cuBLAS / torch):
//   fwd_rir_kernel      RIR partition -> spectrum (both ears packed as one complex signal)
//   fwd_src_kernel      source overlap-save windows -> spectra (cached per clip)
//   mac_ifft_cluster_kernel  N = 4096: mac_bins' per-slot sums over DSMEM into the inverse FFT, emit -> waveform
//   mac_bins_kernel     per-slot partition sums Y (N >= 8192)
//   mac_ifft_kernel     sum_p X[b-p] * H[p] (or Y), inverse FFT, emit the valid half -> waveform
//   spectrogram_kernel  frame + pad + Hann + FFT-512 (ears packed) + |.| + 4x4 mean + log1p
//   audio_conv1_kernel  permute + first Conv2d + ReLU of the policy's AudioCNN
//   audio_encoder_conv_kernel, audio_encoder_linear_kernel   the whole AudioCNN.cnn (conv1-3, then Linear), SAVi's
//                                                            category channels folded into a per-env conv1 bias
//   belief_update_kernel  SAVi's per-env location / category belief update (BeliefPredictor.update)
//   rn_conv_kernel, rn_finish_kernel, brn_maxpool_kernel, rn_head_kernel   SAVi's belief-predictor ResNet-18s
//                                                            (torchvision with BatchNorm, SMT with GroupNorm)
//   smt_fuse_kernel, smt_linear_kernel, smt_attn_kernel, smt_enc_tail_kernel, smt_decoder_kernel   SAVi's scene
//                                                            memory transformer (SMTStateEncoder) on valid tokens
//   smt_transpose_kernel, smt_dec_bwd_kernel, smt_enc_tail_bwd_kernel, smt_attn_bwd_kernel, smt_fuse_bwd_kernel,
//   smt_dw_kernel, smt_reduce_kernel   its backward (PPO update)
//   gru_gemm_kernel, gru_seq_fwd_kernel, gru_seq_bwd_kernel   RNNStateEncoder.seq_forward and its backward (PPO update)
//   cs_gemm_kernel, cs_reduce_kernel, cs_relu_grad_kernel, cs_label_*_kernel   the CNN encoders' conv stack forward and
//                                                            backward in the PPO update (implicit GEMMs across envs)
//   rollout_insert_kernel, rollout_returns_kernel, rollout_gather_kernel   PPO's rollout storage (insert with SAVi's
//                                                            external memory, GAE / returns + advantages, minibatches)
//   frame_gather_kernel remote env workers' RGB / depth frames: bank rows -> float32 observation rows
//   crossfade_kernel, pcm16 kernels
#include <cuda_runtime.h>
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <utility>
#include <vector>

#include "../../include/ssb200.h"
#include "fft16.cuh"
#include "conv64k.cuh"

using namespace ssb;

// Read-once operands (the RIR taps, H in the partition sums, Y in the inverse FFT) are loaded with the
// evict-first policy (__ldcs) so they do not push the re-read data (source spectra, waveform) out of L2.

// ---------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------
#define SSB_MAX_CHUNKS 32
#define SSB_MAX_STREAMS 8
struct TimedLaunch { int kernel; cudaEvent_t a, b; };

struct ssb_ctx {
    int device;
    int sm_count;
    float2* tw[16];      // twiddle tables by log2n (device)
    float2* twm64;       // single-block plan: TWM[r][tau] = w_65536^(tau r), r < 16, tau < 1024
    float* window;       // 512-float centre-padded periodic Hann(400)
    int64_t launches;
    // optional per-kernel CUDA-event timing (bench.py roofline); see ssb_set_kernel_timing
    int timing;
    cudaStream_t s_h2d, s_d2h;                     // copy streams of the pipelined host entry
    cudaEvent_t ev[2 * SSB_MAX_CHUNKS + 2];
    // last two staging buffers written by the copy stream and the event after the kernels that read them
    const void* stage_ptr[2];
    cudaEvent_t stage_done[2];
    int stage_next;
    int64_t last_h2d_bytes, last_d2h_bytes;        // bytes moved by the last ssb_render_batch_host call
    float2* gscratch;                              // [env][9][4096] SH-decode filter spectra
    size_t gscratch_elems;
    float2* yscratch;                              // [env][block][N] partition sums (transposed MAC)
    size_t yscratch_elems;
    float2* nscratch;                              // belief-predictor ResNets: activations and K-range partial sums
    size_t nscratch_elems;
    int* head_ticket;                              // ssb_policy_head_batch: {refused rows, CTAs done}, 0 between calls
    int conv_mode;       // 0: mac_bins + ifft (default), 1: fused mac_ifft
    int n_streams;       // internal compute streams of ssb_render_batch (1 = caller's stream only)
    int n_chunks;        // sub-batches each internal stream works through in turn (L2 footprint, ssb_set_chunks)
    cudaStream_t s_comp[SSB_MAX_STREAMS];
    cudaEvent_t ev_comp[SSB_MAX_STREAMS], ev_fork;
    int debug;           // ssb_set_debug: 32 forces the direct-form SH decode (test hook); 0 in production
    bool attr_sh, attr_shf, attr_shm;   // cudaFuncSetAttribute is per DEVICE: opt-in flags live in the (per-device) context
    // mel filterbanks by (sr, n_mels), built on first use (ssb_logmel_batch)
    struct MelBank { int sr, n_mels; int2* rows; int* ofs; float* w; };
    std::vector<MelBank>* mel;
    // AV-WaN's device maps: pinned staging and device copy of a call's records / poses and tables.  [0] serves
    // ssb_map_update_batch, [1] ssb_map_observe_batch; `done` follows the kernel that last read the buffers.
    struct MapStage { void* h; void* d; size_t cap; cudaEvent_t done; } mstage[2];
    // ssb_rollout_insert_batch: ring of pinned, device-mapped buffers for the sources that arrive on the host;
    // `done` follows the insert kernel that read the slot.
    struct RolloutStage { void* h; void* d; size_t cap; cudaEvent_t done; } rstage[4];
    int rstage_next;
    std::vector<TimedLaunch>* timed;
    char err[512];
};

#define SSB_FAIL(ctx, code, ...)                                  \
    do {                                                          \
        if (ctx) snprintf((ctx)->err, sizeof((ctx)->err), __VA_ARGS__); \
        return (code);                                            \
    } while (0)

#define SSB_CUDA(ctx, call)                                                             \
    do {                                                                                \
        cudaError_t e__ = (call);                                                       \
        if (e__ != cudaSuccess)                                                         \
            SSB_FAIL(ctx, e__ == cudaErrorMemoryAllocation ? SSB_E_OOM : SSB_E_CUDA,    \
                     "%s failed: %s", #call, cudaGetErrorString(e__));                  \
    } while (0)

// Every ABI entry runs on the context's device, whatever the caller's current device is, and restores the
// caller's device afterwards (one process may hold contexts on several devices: per-rank trainers do not, but
// the reference's ``GPU_DEVICE_ID`` / ``TORCH_GPU_ID`` split can put the policy on another device than the renderer).
struct DevGuard {
    int prev = -1, dev;
    explicit DevGuard(int d) : dev(d) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != dev) cudaSetDevice(dev);
    }
    ~DevGuard() { if (prev >= 0 && prev != dev) cudaSetDevice(prev); }
};

// No C++ exception may cross the C ABI (include/ssb200.h: "never throws"): allocating STL containers in an entry
// are wrapped here and reported as SSB_E_OOM / SSB_E_CUDA with a message.
template <class F>
static int abi_call(ssb_ctx* ctx, F&& body) noexcept {
    if (!ctx) return SSB_E_INVALID_ARG;
    try {
        DevGuard g(ctx->device);
        return body();
    } catch (const std::bad_alloc&) {
        snprintf(ctx->err, sizeof(ctx->err), "out of host memory");
        return SSB_E_OOM;
    } catch (...) {
        snprintf(ctx->err, sizeof(ctx->err), "unexpected C++ exception inside libssb200");
        return SSB_E_CUDA;
    }
}

constexpr int kUntimed = -1;  // launch(): a kernel without an SSB_K_* timing slot

// Every kernel launch goes through here: `kernel` enqueues one kernel on `st`.  The launch is counted
// (ssb_launch_count), bracketed by an event pair for ssb_get_kernel_timing when timing is on and `slot` is an SSB_K_*
// index, and its error is returned.
template <class F>
static cudaError_t launch(ssb_ctx* ctx, int slot, cudaStream_t st, F&& kernel) {
    ctx->launches += 1;
    TimedLaunch tl{slot, nullptr, nullptr};
    bool timed = slot != kUntimed && ctx->timing && ctx->timed;
    if (timed && cudaEventCreate(&tl.a) != cudaSuccess) timed = false;
    if (timed && cudaEventCreate(&tl.b) != cudaSuccess) { cudaEventDestroy(tl.a); timed = false; }
    if (timed) cudaEventRecord(tl.a, st);
    kernel();
    const cudaError_t e = cudaGetLastError();
    if (timed) {
        cudaEventRecord(tl.b, st);
        try {                                     // the kernel is already queued: drop the sample rather than fail
            ctx->timed->push_back(tl);
        } catch (...) {
            cudaEventDestroy(tl.a);
            cudaEventDestroy(tl.b);
        }
    }
    return e;
}

// ---------------------------------------------------------------------------
// forward FFT kernels
// ---------------------------------------------------------------------------
template <int LOG2N>
__device__ __forceinline__ void store_slots(float2* __restrict__ dst, const float2 (&v)[16], int t) {
    constexpr int T = FftPlan<LOG2N>::T;
#pragma unroll
    for (int i = 0; i < 16; ++i) dst[i * T + t] = v[i];
}

// copy the twiddle rows of passes >= 1 into shared memory (a few hundred float2)
template <int LOG2N>
__device__ __forceinline__ void stage_small_twiddles(float2* __restrict__ stw, const float2* __restrict__ tw, int t) {
    using P = FftPlan<LOG2N>;
    for (int i = t; i < P::TW_SMALL_ELEMS; i += P::T) stw[i] = __ldg(tw + P::TW_SMALL_OFFSET + i);
}

// grid (max_parts * n_terms, B); block T.  H[env][term][p][N] in slot order.
template <int LOG2N>
__global__ void __launch_bounds__(FftPlan<LOG2N>::T)
fwd_rir_kernel(const ssb_req* __restrict__ reqs, const float2* __restrict__ rir_bank,
               float2* __restrict__ H, int max_parts, long long h_elems_per_env,
               const float2* __restrict__ tw) {
    using P = FftPlan<LOG2N>;
    extern __shared__ float2 smem[];
    float2* stw = smem + P::SMEM_ELEMS;
    constexpr int PART = P::N / 2;
    const int env = blockIdx.y;
    const int term = blockIdx.x / max_parts;
    const int p = blockIdx.x % max_parts;
    const ssb_req& rq = reqs[env];
    if (rq.flags & SSB_FLAG_SILENT) return;
    const int taps = rq.term[term].rir_taps;
    if (p * PART >= taps) return;                      // this partition is never read
    const int t = threadIdx.x;
    const float2* __restrict__ src = rir_bank + rq.term[term].rir_offset;
    float2 v[16];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        int n = p * PART + t + q * P::T;
        v[q] = n < taps ? __ldcs(src + n) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int q = 8; q < 16; ++q) v[q] = make_float2(0.f, 0.f);
    const Tw6 w0 = load_tw6<true>(tw, P::T, t);
    stage_small_twiddles<LOG2N>(stw, tw, t);           // visible after the first exchange barrier
    fft_forward<LOG2N>(v, t, smem, w0, stw);
    float2* dst = H + (long long)env * h_elems_per_env + ((long long)term * max_parts + p) * P::N;
    store_slots<LOG2N>(dst, v, t);
}

// grid (nw); block T.  X[j][N] in slot order; window j covers samples
// [m0 + (j - wofs - 1) P, m0 + (j - wofs + 1) P).
template <int LOG2N>
__global__ void __launch_bounds__(FftPlan<LOG2N>::T)
fwd_src_kernel(const float* __restrict__ src, int S, long long m0, int wrap, int wofs,
               float2* __restrict__ X, const float2* __restrict__ tw) {
    using P = FftPlan<LOG2N>;
    extern __shared__ float2 smem[];
    float2* stw = smem + P::SMEM_ELEMS;
    constexpr int PART = P::N / 2;
    const int j = blockIdx.x;
    const int t = threadIdx.x;
    const Tw6 w0 = load_tw6<true>(tw, P::T, t);
    stage_small_twiddles<LOG2N>(stw, tw, t);
    const long long base = m0 + (long long)(j - wofs - 1) * PART;
    float2 v[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) {
        long long n = base + t + q * P::T;
        float x = 0.f;
        if (n >= 0) {
            if (n < S) x = __ldg(src + n);
            else if (wrap && n - S < S) x = __ldg(src + (n - S));
        }
        v[q] = make_float2(x, 0.f);
    }
    fft_forward<LOG2N>(v, t, smem, w0, stw);
    store_slots<LOG2N>(X + (long long)j * P::N, v, t);
}

// ---------------------------------------------------------------------------
// "transposed" multiply-accumulate: one thread per (env, spectrum slot) forms ALL the block sums
//   Y[b][s] = sum_p X[b - p + wofs][s] * H[p][s]
// so every H value crosses the L2->SM link once (the fused loop in mac_ifft_kernel re-reads each
// partition for every block: 4.9 MB per env at config 2 against 0.26 + 0.70 MB here); repeated
// touches of the same slot column are L1 hits.  grid (N / 256, B); block 256.
// ---------------------------------------------------------------------------
template <int LOG2N, int NPMAX, int NBMAX>
__global__ void __launch_bounds__(256)
mac_bins_kernel(const ssb_req* __restrict__ reqs, const float2* __restrict__ xpool, const float2* __restrict__ H,
                int max_parts, int n_terms, long long h_elems_per_env, float2* __restrict__ Y, int n_blocks, int sr) {
    using P = FftPlan<LOG2N>;
    constexpr int PART = P::N / 2;
    const int env = blockIdx.y;
    const int s = blockIdx.x * 256 + threadIdx.x;
    const ssb_req& rq = reqs[env];
    if (rq.flags & SSB_FLAG_SILENT) return;
    const int nvalid = min(rq.out_samples, sr);
    const int nblk = (nvalid + PART - 1) / PART;
    float2* __restrict__ yo = Y + (long long)env * n_blocks * P::N + s;
    bool first = true;                                          // first term stores, later terms accumulate into Y
    for (int term = 0; term < n_terms; ++term) {
        const ssb_conv_term& ct = rq.term[term];
        if (ct.rir_taps <= 0) continue;
        const int nparts = min((ct.rir_taps + PART - 1) / PART, max_parts);
        const float2* __restrict__ hp = H + (long long)env * h_elems_per_env + (long long)term * max_parts * P::N + s;
        const float2* __restrict__ xp = xpool + ct.x_offset + s;
        if (ct.x_wofs == 0 && nparts <= NPMAX && nblk <= NBMAX && ct.x_nw >= nblk) {
            // fast path (clip starts at offset 0): every operand is loaded exactly once, up front
            float2 h[NPMAX], x[NBMAX];
#pragma unroll
            for (int p = 0; p < NPMAX; ++p) h[p] = p < nparts ? __ldcs(hp + (long long)p * P::N) : make_float2(0.f, 0.f);
#pragma unroll
            for (int w = 0; w < NBMAX; ++w) x[w] = w < nblk ? __ldg(xp + (long long)w * P::N) : make_float2(0.f, 0.f);
#pragma unroll
            for (int b = 0; b < NBMAX; ++b) {
                if (b < nblk) {
                    // x * h = x.x * h + i * (x.y * h): two accumulators, ONE swizzled add at the end, so the
                    // inner loop is four FFMA per complex multiply-accumulate with no operand shuffling
                    float2 acc_re = first ? make_float2(0.f, 0.f) : yo[(long long)b * P::N];
                    float2 acc_im = make_float2(0.f, 0.f);
#pragma unroll
                    for (int p = 0; p < NPMAX; ++p) {
                        if (p <= b) {                            // window b - p >= 0; h[p] is 0 beyond nparts
                            acc_re = fma2(bcast(x[b - p].x), h[p], acc_re);
                            acc_im = fma2(bcast(x[b - p].y), h[p], acc_im);
                        }
                    }
                    yo[(long long)b * P::N] = add2(acc_re, make_float2(-acc_im.y, acc_im.x));
                }
            }
        } else {
            // general path: arbitrary window offset / partition count; repeated touches are L1 hits
            for (int b = 0; b < nblk; ++b) {
                float2 acc = first ? make_float2(0.f, 0.f) : yo[(long long)b * P::N];
                const int p_lo = max(0, b + ct.x_wofs - (ct.x_nw - 1));
                const int p_hi = min(nparts - 1, b + ct.x_wofs);
                for (int p = p_lo; p <= p_hi; ++p) {
                    const float2 h = hp[(long long)p * P::N];
                    const float2 x = __ldg(xp + (long long)(b - p + ct.x_wofs) * P::N);
                    acc = cfma(x, h, acc);
                }
                yo[(long long)b * P::N] = acc;
            }
        }
        first = false;
    }
    if (first)                                                  // no term had taps: the inverse-FFT kernel writes zeros itself
        return;
}

// ---------------------------------------------------------------------------
// Default schedule at N = 4096: mac_bins_kernel's partition sums, inverse FFT and emit for one env per cluster of
// CL CTAs, with the sums kept on chip.  Rank k owns the slot rows i in [k 16/CL, (k+1) 16/CL): for each of its slots
// s = i T + t a thread forms the sums Y[b][s] of EVERY block with exactly mac_bins_kernel's arithmetic (same paths,
// same term order), and stores each over distributed shared memory into rank b % CL, which inverse-transforms its
// blocks b = k, k + CL, ... from its own shared memory: Y never reaches L2 or HBM (92 MB of writes and as many reads
// per config-2 step).  The receive buffer of a block, [i][t] in a FftPlan::SMEM_ELEMS region, doubles as that
// block's FFT exchange buffer.  A CTA holds `lbr` such buffers (host: mac_round_blocks); more blocks per CTA run in
// rounds.
//
// No hang by construction: the early exits (silent env, no term with taps) and the round count depend only on the
// env's request, which every rank of the cluster reads, so either every CTA reaches each cluster barrier or none
// does.  Blocks past the rendered window are zero-filled after the barriers, not instead of them.
// grid (CL * B), cluster (CL, 1, 1), block T, dynamic shared memory lbr * SMEM_ELEMS float2.
// ---------------------------------------------------------------------------
template <int LOG2N, int CL>
__global__ void __launch_bounds__(FftPlan<LOG2N>::T, 2)
mac_ifft_cluster_kernel(const ssb_req* __restrict__ reqs, const float2* __restrict__ xpool, const float2* __restrict__ H,
                        int max_parts, int n_terms, long long h_elems_per_env, int n_blocks, int lbr,
                        float* __restrict__ wave, long long wave_stride, int sr, const float2* __restrict__ tw) {
    using P = FftPlan<LOG2N>;
    constexpr int NPMAX = 8, NBMAX = 24;                        // mac_bins_kernel<LOG2N, 8, 24>'s fast-path limits
    constexpr int ROWS = 16 / CL;
    constexpr int PART = P::N / 2;
    static_assert(CL == 1 || CL == 2 || CL == 4 || CL == 8, "cluster size");
    extern __shared__ float2 smem[];
    cg::cluster_group cluster = cg::this_cluster();
    const int k = (int)cluster.block_rank();
    const int env = blockIdx.x / CL;
    const int t = threadIdx.x;
    const ssb_req& rq = reqs[env];
    float* __restrict__ wl = wave + (long long)env * 2 * wave_stride;
    float* __restrict__ wr = wl + wave_stride;
    const int nvalid = (rq.flags & SSB_FLAG_SILENT) ? 0 : min(rq.out_samples, sr);
    bool any = false;
    for (int term = 0; term < n_terms; ++term) any |= rq.term[term].rir_taps > 0;
    const int nblk = any ? max(0, (nvalid + PART - 1) / PART) : 0;     // blocks with sums: b < nblk
    const int n_rounds = ((nblk + CL - 1) / CL + lbr - 1) / lbr;
    // Round 0 needs every peer running before the first store into its shared memory, not before the first loads: the
    // CTA arrives on entry and waits (join) once its first slot row's operand loads are in flight, so their latency
    // overlaps the wait for the other CTAs of the cluster.  Every thread joins exactly once, before any DSMEM access.
    // The arrive is relaxed: this CTA has written nothing yet, so there is nothing to release (a release arrive would
    // first wait for the request loads in flight).  launch_mac_ifft_cluster always sets the cluster dimension (CL = 1
    // too), so cluster.barrier_wait() is the cluster barrier's wait that pairs with this arrive.
    bool joined = n_rounds == 0;
    if (!joined) asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
    auto join = [&] {
        if (!joined) { cluster.barrier_wait(); joined = true; }
    };
    for (int r = 0; r < n_rounds; ++r) {
        if (r > 0) cluster.sync();                              // peers' buffers of the last round are free
        // this round: blocks [b_lo, b_hi); block b goes to rank b % CL, buffer b / CL - r lbr
        const int b_lo = r * lbr * CL, b_hi = min(nblk, (r + 1) * lbr * CL);
#pragma unroll 1
        for (int ii = 0; ii < ROWS; ++ii) {
            const int s = (k * ROWS + ii) * P::T + t;
            float2* const ybase = smem - r * lbr * P::SMEM_ELEMS + s;
            bool first = true;                                  // first term stores, later terms accumulate into Y
            for (int term = 0; term < n_terms; ++term) {
                const ssb_conv_term& ct = rq.term[term];
                if (ct.rir_taps <= 0) continue;
                const int nparts = min((ct.rir_taps + PART - 1) / PART, max_parts);
                const float2* __restrict__ hp = H + (long long)env * h_elems_per_env + (long long)term * max_parts * P::N + s;
                const float2* __restrict__ xp = xpool + ct.x_offset + s;
                if (ct.x_wofs == 0 && nparts <= NPMAX && nblk <= NBMAX && ct.x_nw >= nblk) {
                    // fast path (clip starts at offset 0): every operand is loaded exactly once, up front
                    float2 h[NPMAX], x[NBMAX];
#pragma unroll
                    for (int p = 0; p < NPMAX; ++p) h[p] = p < nparts ? __ldcs(hp + (long long)p * P::N) : make_float2(0.f, 0.f);
#pragma unroll
                    for (int w = 0; w < NBMAX; ++w) x[w] = w < b_hi ? __ldg(xp + (long long)w * P::N) : make_float2(0.f, 0.f);
                    join();
#pragma unroll
                    for (int b = 0; b < NBMAX; ++b) {
                        if (b >= b_lo && b < b_hi) {
                            float2* y = cluster.map_shared_rank(ybase + (b / CL) * P::SMEM_ELEMS, b % CL);
                            float2 acc_re = first ? make_float2(0.f, 0.f) : *y;
                            float2 acc_im = make_float2(0.f, 0.f);
#pragma unroll
                            for (int p = 0; p < NPMAX; ++p) {
                                if (p <= b) {
                                    acc_re = fma2(bcast(x[b - p].x), h[p], acc_re);
                                    acc_im = fma2(bcast(x[b - p].y), h[p], acc_im);
                                }
                            }
                            *y = add2(acc_re, make_float2(-acc_im.y, acc_im.x));
                        }
                    }
                } else {
                    join();
                    for (int b = b_lo; b < b_hi; ++b) {
                        float2* y = cluster.map_shared_rank(ybase + (b / CL) * P::SMEM_ELEMS, b % CL);
                        float2 acc = first ? make_float2(0.f, 0.f) : *y;
                        const int p_lo = max(0, b + ct.x_wofs - (ct.x_nw - 1));
                        const int p_hi = min(nparts - 1, b + ct.x_wofs);
                        for (int p = p_lo; p <= p_hi; ++p) {
                            const float2 h = hp[(long long)p * P::N];
                            const float2 x = __ldg(xp + (long long)(b - p + ct.x_wofs) * P::N);
                            acc = cfma(x, h, acc);
                        }
                        *y = acc;
                    }
                }
                first = false;
            }
        }
        join();                                                 // (a round always has a term with taps: joined already)
        cluster.sync();                                         // every sum of this round is in its receive buffer
        for (int lb = 0; lb < lbr; ++lb) {
            const int b = (r * lbr + lb) * CL + k;
            if (b >= nblk) break;
            float2* __restrict__ buf = smem + lb * P::SMEM_ELEMS;
            float2 acc[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[i] = buf[i * P::T + t];
            __syncthreads();                                    // the FFT's first exchange overwrites the buffer
            fft_inverse<LOG2N>(acc, t, buf, tw, tw + P::TW_SMALL_OFFSET);
            constexpr float scale = 1.0f / (float)P::N;
            const int n0 = b * PART;
#pragma unroll
            for (int q = 8; q < 16; ++q) {
                int n = n0 + t + (q - 8) * P::T;
                if (n < sr) {
                    bool ok = n < nvalid;
                    wl[n] = ok ? acc[q].x * scale : 0.f;
                    wr[n] = ok ? acc[q].y * scale : 0.f;
                }
            }
        }
    }
    for (int b = k; b < n_blocks; b += CL) {                    // silent / past the rendered window / zero RIR
        if (b < nblk) continue;
        const int n0 = b * PART;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            int n = n0 + t + q * P::T;
            if (n < sr) { wl[n] = 0.f; wr[n] = 0.f; }
        }
    }
}

// ---------------------------------------------------------------------------
// multiply-accumulate over partitions + inverse FFT + emit
// grid (B, n_blocks); block T.  The explicit minimum of one CTA per SM is not a no-op: without it ptxas caps the
// N = 8192 instances at 64 registers.
// ---------------------------------------------------------------------------
template <int LOG2N, bool FROM_Y>
__global__ void __launch_bounds__(FftPlan<LOG2N>::T, 1)
mac_ifft_kernel(const ssb_req* __restrict__ reqs, const float2* __restrict__ xpool,
                const float2* __restrict__ H, int max_parts, int n_terms, long long h_elems_per_env,
                float* __restrict__ wave, long long wave_stride, int sr, const float2* __restrict__ tw) {
    using P = FftPlan<LOG2N>;
    extern __shared__ float2 smem[];
    constexpr int PART = P::N / 2;
    // env is the fastest block index: CTAs resident together work on the same block b of different
    // envs and read the same source windows X[b-p] (one L2->L1 fill serves both)
    const int env = blockIdx.x;
    const int b = blockIdx.y;
    const int t = threadIdx.x;
    const ssb_req& rq = reqs[env];
    float* __restrict__ wl = wave + (long long)env * 2 * wave_stride;
    float* __restrict__ wr = wl + wave_stride;
    const int n0 = b * PART;
    const int nvalid = (rq.flags & SSB_FLAG_SILENT) ? 0 : min(rq.out_samples, sr);
    bool any = false;
    if (n0 < nvalid) {
        for (int term = 0; term < n_terms; ++term) any |= rq.term[term].rir_taps > 0;
    }
    if (!any) {                                        // silent / past the rendered window / zero RIR
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            int n = n0 + t + q * P::T;
            if (n < sr) { wl[n] = 0.f; wr[n] = 0.f; }
        }
        return;
    }
    float2 acc[16];
    if constexpr (FROM_Y) {
        // the partition sums were formed per bin by mac_bins_kernel; H here is its output Y[env][b][N]
        const float2* __restrict__ yp = H + ((long long)env * gridDim.y + b) * P::N + t;
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[i] = __ldcs(yp + i * P::T);
    } else {
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = make_float2(0.f, 0.f);
    for (int term = 0; term < n_terms; ++term) {
        const ssb_conv_term& ct = rq.term[term];
        if (ct.rir_taps <= 0) continue;
        const int nparts = min((ct.rir_taps + PART - 1) / PART, max_parts);
        const float2* __restrict__ Hb = H + (long long)env * h_elems_per_env + (long long)term * max_parts * P::N;
        const float2* __restrict__ Xb = xpool + ct.x_offset;
        // window index j = b - p + wofs must lie in [0, nw)
        int p_lo = max(0, b + ct.x_wofs - (ct.x_nw - 1));
        int p_hi = min(nparts - 1, b + ct.x_wofs);
        for (int p = p_lo; p <= p_hi; ++p) {
            const float2* __restrict__ hp = Hb + (long long)p * P::N + t;
            const float2* __restrict__ xp = Xb + (long long)(b - p + ct.x_wofs) * P::N + t;
            float2 h[16], x[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) { h[i] = hp[i * P::T]; x[i] = __ldg(xp + i * P::T); }
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[i] = cfma(x[i], h[i], acc[i]);
        }
    }
    }
    // the later passes read their twiddles straight from the (L1-resident) global table, as the STFT kernel does,
    // so no block barrier is spent staging them in shared memory
    fft_inverse<LOG2N>(acc, t, smem, tw, tw + P::TW_SMALL_OFFSET);
    constexpr float scale = 1.0f / (float)P::N;
#pragma unroll
    for (int q = 8; q < 16; ++q) {
        int n = n0 + t + (q - 8) * P::T;
        if (n < sr) {
            bool ok = n < nvalid;
            wl[n] = ok ? acc[q].x * scale : 0.f;
            wr[n] = ok ? acc[q].y * scale : 0.f;
        }
    }
}

// ---------------------------------------------------------------------------
// spectrogram: one warp per POOLED COLUMN (4 consecutive STFT frames), warps fully independent
// (only __syncwarp): frame + pad + Hann + packed FFT-512 + |.| per ear, magnitudes accumulated
// over the 4 frames in registers, pooled over 4 bins with two shuffles, log1p, store.
// ---------------------------------------------------------------------------
constexpr int SPEC_BUF = 512 + 32;

// sqrt.approx.ftz.f32: one MUFU, max relative error 2^-23 (IEEE sqrtf expands to ~8 instructions, the
// non-ftz approx form to 4: range test + two scalings around the MUFU for denormal inputs)
__device__ __forceinline__ float fast_sqrt(float x) {
    float y;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ int nat_idx(int k) { return k + ((k >> 8) << 3); }   // de-conflict k and 256+k

// Samples: element idx = lane + 32 q of frame f is sample 160 f + idx - 256, and 160 = 5 * 32, so
// over the 4 frames of a column lane `lane` only ever touches x_j = y[n0 + lane + 32 j], j = 1..29
// (frame fr uses j = q + 5 fr): each frame needs just 5 new samples per ear; they are fetched
// before the previous frame's FFT and shifted into a 14-deep register window.
template <bool REFLECT, bool INTERIOR>
__device__ __forceinline__ float spec_sample(const float* __restrict__ y, int n, int sr) {
    if (INTERIOR) return __ldg(y + n);
    if (REFLECT) {                       // np.pad(y, 256, mode='reflect'): librosa < 0.10
        if (n < 0) n = -n;
        if (n >= sr) n = 2 * (sr - 1) - n;
        n = max(0, min(n, sr - 1));      // only reached by frames past the end (weight 0)
        return __ldg(y + n);
    }
    return (n >= 0 && n < sr) ? __ldg(y + n) : 0.f;   // mode='constant': librosa >= 0.10
}

// One pooled column (4 frames) by one warp.  INTERIOR: every sample in range and all 4 frames real.
// Everything that does not change from frame to frame -- both passes' twiddles, the lane's 14 window weights and
// its exchange addresses -- is set up once per column, outside the frame loop.
template <bool REFLECT, bool INTERIOR>
__device__ __forceinline__ void spec_column(const float* __restrict__ yl, const float* __restrict__ yr, int sr,
                                            int n_frames, int col, int lane, float2* __restrict__ buf,
                                            const float2* __restrict__ stw, const float* __restrict__ swin,
                                            float (&accl)[8], float (&accr)[8], float& acc64l, float& acc64r) {
    const Tw6 w0 = load_tw6<true>(stw, 32, lane);
    constexpr int st1 = FftPlan<9>::stride(1);
    const Tw6 w1 = load_tw6<true>(stw + FftPlan<9>::TW_SMALL_OFFSET, st1, lane % st1);
    // centre-padded Hann: 0 for idx < 56, idx >= 456.  Edge columns read it per frame: holding it too would take that
    // path past the 128 registers of 16 warps per SM and spill.
    float win[15];
#pragma unroll
    for (int q = 1; q < 15; ++q) win[q] = INTERIOR ? __ldg(swin + lane + 32 * q) : 0.f;
    const int n0 = col * SSB_POOL * SSB_HOP - SSB_N_FFT / 2 + lane;          // sample of x_0 for this lane
    // interior columns: every sample is a fixed offset from these two pointers, which advance by one hop per frame
    const float* __restrict__ pl = yl + n0;
    const float* __restrict__ pr = yr + n0;
    float2 x[15];                                                            // window of the current frame: (L, R) pairs, q = 1..14
#pragma unroll
    for (int q = 1; q < 15; ++q) {
        if (INTERIOR) x[q] = make_float2(__ldg(pl + 32 * q), __ldg(pr + 32 * q));
        else x[q] = make_float2(spec_sample<REFLECT, false>(yl, n0 + 32 * q, sr), spec_sample<REFLECT, false>(yr, n0 + 32 * q, sr));
    }
    // After the FFT, lane 2a holds P_a[i] and lane 2a+1 holds Q_a[i] for kap = a + 16 i (the last radix-2 stage, across
    // lane pairs, is folded into the reads below: Z[kap] = P[kap] + Q[kap], Z[kap + 256] = P[kap] - Q[kap]).  Stored at
    // float2 lane + 32 i = 2 kap + (lane & 1), float4 kap of buf is {P[kap], Q[kap]}: one LDS.128 per bin, conflict free.
    const float4* __restrict__ pq = reinterpret_cast<const float4*>(buf);
    const float4* __restrict__ pq_k = pq + lane;                             // bin k = lane + 32 m at pq_k[32 m]
    const float4* __restrict__ pq_kk = pq + (256 - lane);                    // bin 256 - k at pq_kk[-32 m], m >= 1
    const float4* __restrict__ pq_kk0 = pq + ((256 - lane) & 255);           // m = 0: bin 0 for lane 0
#pragma unroll 1
    for (int fr = 0; fr < SSB_POOL; ++fr) {
        // prefetch the 5 new samples of the next frame (j = 15 + 5 fr ..); latency hides behind this frame's FFT
        float2 nx[5];
#pragma unroll
        for (int u = 0; u < 5; ++u) {
            const int j = 15 + u;
            if (INTERIOR) nx[u] = fr + 1 < SSB_POOL ? make_float2(__ldg(pl + 32 * j), __ldg(pr + 32 * j)) : make_float2(0.f, 0.f);
            else nx[u] = fr + 1 < SSB_POOL ? make_float2(spec_sample<REFLECT, false>(yl, n0 + 32 * (j + 5 * fr), sr),
                                                         spec_sample<REFLECT, false>(yr, n0 + 32 * (j + 5 * fr), sr))
                                           : make_float2(0.f, 0.f);
        }
        const bool f_ok = INTERIOR || (col * SSB_POOL + fr < n_frames);     // frames past the end add 0 (block_reduce pads with 0)
        float2 v[16];
        v[0] = make_float2(0.f, 0.f);                          // idx < 56 and idx >= 456 lie outside the 400-tap window
        v[15] = make_float2(0.f, 0.f);
#pragma unroll
        for (int q = 1; q < 15; ++q) v[q] = mul2(bcast(INTERIOR ? win[q] : f_ok ? __ldg(swin + lane + 32 * q) : 0.f), x[q]);
        fft_forward<9, false>(v, lane, buf, w0, w1);
        __syncwarp();
#pragma unroll
        for (int i = 0; i < 16; ++i) buf[lane + 32 * i] = v[i];
        __syncwarp();
        // Z = FFT(w*(yL + i yR)):  XL[k] = (Z[k] + conj Z[N-k])/2,  XR[k] = (Z[k] - conj Z[N-k])/(2i);
        // for 0 < k < 256: Z[N-k] = Z[(256-k) + 256] = P[256-k] - Q[256-k]; Z[N-0] = Z[0]
        float4 pq0;
#pragma unroll
        for (int m = 0; m < 8; ++m) {
            const float4 ck = pq_k[32 * m];
            const float4 ckk = m == 0 ? pq_kk0[0] : pq_kk[-32 * m];
            if (m == 0) pq0 = ck;
            const float2 a = add2(make_float2(ck.x, ck.y), make_float2(ck.z, ck.w));
            float2 bb;
            if (m == 0) bb = fma2(bcast(lane == 0 ? 1.f : -1.f), make_float2(ckk.z, ckk.w), make_float2(ckk.x, ckk.y));
            else bb = sub2(make_float2(ckk.x, ckk.y), make_float2(ckk.z, ckk.w));
            const float2 cb = make_float2(bb.x, -bb.y);
            const float2 l = add2(a, cb), r = sub2(a, cb);     // A + conj(B), A - conj(B)
            const float2 l2 = mul2(l, l), r2 = mul2(r, r);
            accl[m] += fast_sqrt(l2.x + l2.y);
            accr[m] += fast_sqrt(r2.x + r2.y);
        }
        if (lane == 0) {                                       // bin 256 = P[0] - Q[0] is alone in pooled row 64
            const float2 a = sub2(make_float2(pq0.x, pq0.y), make_float2(pq0.z, pq0.w));
            acc64l += fabsf(a.x);
            acc64r += fabsf(a.y);
        }
        __syncwarp();                                          // buf is rewritten by the next frame's exchange
        // slide the sample window by one hop (5 x 32 samples)
#pragma unroll
        for (int q = 1; q < 10; ++q) x[q] = x[q + 5];
#pragma unroll
        for (int u = 0; u < 5; ++u) x[10 + u] = nx[u];
        pl += SSB_HOP;
        pr += SSB_HOP;
    }
}

// grid (cols, B); block = ONE warp.  Everything that selects a code path (column index, interior
// test) derives from blockIdx, so the compiler can prove the warp converged and the shuffles and
// __syncwarp()s stay single instructions (with several warps per CTA and a per-warp column they
// were compiled into WARPSYNC.COLLECTIVE sequences).
// Registers: the sample window, the prefetch, the 18 accumulators, the 16 FFT points, both passes' twiddles and the
// window weights fit the 128 of 16 resident warps per SM with no spills (16 warps run the kernel about 9 % faster than the
// 15 that 135 registers allow).  Keep it unspilled: spills cost more, mostly in L1/L2 traffic shared with the
// convolution kernels on the other stream, than the extra warps gain.
template <bool REFLECT>
__global__ void __launch_bounds__(32, 16)
spectrogram_kernel(const float* __restrict__ wave, long long wave_stride, int sr, int n_frames, int cols,
                   float* __restrict__ out, const float2* __restrict__ tw,
                   const float* __restrict__ window, int nchw, const ssb_req* __restrict__ reqs, int n_terms) {
    __shared__ __align__(16) float2 xbuf[SPEC_BUF];
    const int lane = threadIdx.x;
    const int col = blockIdx.x;
    const int env = blockIdx.y;
    const float* __restrict__ yl = wave + (long long)env * 2 * wave_stride;
    const float* __restrict__ yr = yl + wave_stride;
    // every x_j, j = 1..29, in range and all four frames real => no padding logic at all
    const int first = col * SSB_POOL * SSB_HOP - SSB_N_FFT / 2;
    const bool interior = first + 32 >= 0 && first + 32 * 30 <= sr && col * SSB_POOL + SSB_POOL <= n_frames;
    float accl[8], accr[8], acc64l = 0.f, acc64r = 0.f;
#pragma unroll
    for (int m = 0; m < 8; ++m) { accl[m] = 0.f; accr[m] = 0.f; }
    // With the render requests (reqs != null), an env the convolution left all zero -- silent, no term with taps, or
    // nothing to output -- skips the transforms: on a zero waveform they would only add +0 to the accumulators.
    bool dead = false;
    if (reqs) {
        const ssb_req& rq = reqs[env];
        bool any = false;
        for (int term = 0; term < n_terms; ++term) any |= rq.term[term].rir_taps > 0;
        dead = (rq.flags & SSB_FLAG_SILENT) || rq.out_samples <= 0 || !any;
    }
    if (!dead && interior)
        spec_column<REFLECT, true>(yl, yr, sr, n_frames, col, lane, xbuf, tw, window, accl, accr, acc64l, acc64r);
    else if (!dead)
        spec_column<REFLECT, false>(yl, yr, sr, n_frames, col, lane, xbuf, tw, window, accl, accr, acc64l, acc64r);
    // pool 4 adjacent bins (lanes): after the two xor-shuffles every lane of a 4-lane group holds the group sum;
    // lane q of the group then finishes rows m = 2q, 2q+1 only (4 log1p per lane instead of 16).
    // scale: 0.5 (ear packing) / 16 (4x4 mean)
    const int q = lane & 3;
    float ml[2] = {0.f, 0.f}, mr[2] = {0.f, 0.f};
#pragma unroll
    for (int m = 0; m < 8; ++m) {
        float l = accl[m], r = accr[m];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        r += __shfl_xor_sync(0xffffffffu, r, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        r += __shfl_xor_sync(0xffffffffu, r, 2);
        if (q == (m >> 1)) { ml[m & 1] = l; mr[m & 1] = r; }
    }
    const float v64l = log1pf(acc64l * (1.0f / 16.0f)), v64r = log1pf(acc64r * (1.0f / 16.0f));
    if (!nchw) {
        // reference layout (65, T', 2): ears interleaved (nav.py:98 np.stack(axis=-1))
        float* __restrict__ o = out + (((long long)env * SSB_SPEC_ROWS) * cols + col) * 2;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int row = (lane >> 2) + 8 * (2 * q + j);
            *reinterpret_cast<float2*>(o + (long long)row * cols * 2) =
                make_float2(log1pf(ml[j] * (0.5f / 16.0f)), log1pf(mr[j] * (0.5f / 16.0f)));
        }
        if (lane == 0) *reinterpret_cast<float2*>(o + (long long)64 * cols * 2) = make_float2(v64l, v64r);
    } else {
        // channels-first (2, 65, T'): what AudioCNN's permute(0, 3, 1, 2) produces (audio_cnn.py:86)
        float* __restrict__ ol = out + ((long long)env * 2 * SSB_SPEC_ROWS) * cols + col;
        float* __restrict__ orr = ol + (long long)SSB_SPEC_ROWS * cols;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int row = (lane >> 2) + 8 * (2 * q + j);
            ol[(long long)row * cols] = log1pf(ml[j] * (0.5f / 16.0f));
            orr[(long long)row * cols] = log1pf(mr[j] * (0.5f / 16.0f));
        }
        if (lane == 0) { ol[(long long)64 * cols] = v64l; orr[(long long)64 * cols] = v64r; }
    }
}


// ---------------------------------------------------------------------------
// log-mel spectrogram.  EXTENSION: BASELINE.json configs[2] and the north star name a log-mel front end, the
// reference itself has none (SURVEY.md 8(d)); defined here as
//     out[env][j][t][ear] = log1p( sum_k M[j][k] * |STFT(wave[env][ear])[k][t]|^power ),   power in {1, 2},
// with the reference's STFT (n_fft 512, hop 160, Hann(400), centre padding: nav.py:89-92) and M the Slaney
// mel filterbank of librosa.filters.mel(sr, 512, n_mels) (area-normalised triangles, fmin 0, fmax sr/2), i.e.
// log1p(librosa.feature.melspectrogram(...)) -- the same log1p compression the reference applies (nav.py:97).
// One warp per group of 4 consecutive frames (the sample window slides exactly as in spec_column).  The
// filterbank is a sparse matrix -- every bin feeds at most two triangles, 2 * 257 non-zeros in all against
// 64 * 257 = 16448 dense entries -- so it is applied as per-mel sparse dot products from shared memory; a dense
// tensor-core GEMM would first have to write the (257, T) power spectra to HBM (2 x 284 KB per env at
// 44.1 kHz, more than every other byte this path moves) to do 32x the arithmetic.
// ---------------------------------------------------------------------------
constexpr int MEL_MAX = 64;                  // two mel rows per lane
constexpr int MEL_PBUF = SSB_N_FFT / 2 + 1;  // 257 bins

template <bool REFLECT>
__global__ void __launch_bounds__(32, 16)
logmel_kernel(const float* __restrict__ wave, long long wave_stride, int sr, int n_frames, int n_mels, int power,
              float* __restrict__ out, const float2* __restrict__ tw, const float* __restrict__ window,
              const int2* __restrict__ mel_rows /* (first bin, count) */, const int* __restrict__ mel_ofs,
              const float* __restrict__ mel_w) {
    __shared__ float2 buf[SPEC_BUF];
    __shared__ float2 pbuf[MEL_PBUF + 1];
    const int lane = threadIdx.x;
    const int t0 = blockIdx.x * SSB_POOL;                       // first frame of this warp
    const int env = blockIdx.y;
    const float* __restrict__ yl = wave + (long long)env * 2 * wave_stride;
    const float* __restrict__ yr = yl + wave_stride;
    const Tw6 w0 = load_tw6<true>(tw, 32, lane);
    const int n0 = t0 * SSB_HOP - SSB_N_FFT / 2 + lane;
    float2 x[15];
#pragma unroll
    for (int q = 1; q < 15; ++q)
        x[q] = make_float2(spec_sample<REFLECT, false>(yl, n0 + 32 * q, sr), spec_sample<REFLECT, false>(yr, n0 + 32 * q, sr));
    // this lane's mel rows j = lane and lane + 32
    int2 row[2];
    const float* __restrict__ wrow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int j = lane + 32 * h;
        row[h] = j < n_mels ? __ldg(mel_rows + j) : make_int2(0, 0);
        wrow[h] = mel_w + (j < n_mels ? __ldg(mel_ofs + j) : 0);
    }
    float2 res[2][SSB_POOL];
#pragma unroll 1
    for (int fr = 0; fr < SSB_POOL; ++fr) {
        float2 nx[5];
#pragma unroll
        for (int u = 0; u < 5; ++u) {
            const int n = n0 + 32 * (15 + 5 * fr + u);
            nx[u] = fr + 1 < SSB_POOL ? make_float2(spec_sample<REFLECT, false>(yl, n, sr), spec_sample<REFLECT, false>(yr, n, sr))
                                      : make_float2(0.f, 0.f);
        }
        float2 v[16];
        v[0] = make_float2(0.f, 0.f);
        v[15] = make_float2(0.f, 0.f);
#pragma unroll
        for (int q = 1; q < 15; ++q) v[q] = mul2(bcast(__ldg(window + lane + 32 * q)), x[q]);
        fft_forward<9>(v, lane, buf, w0, tw + FftPlan<9>::TW_SMALL_OFFSET);
        __syncwarp();
#pragma unroll
        for (int i = 0; i < 16; ++i) buf[nat_idx((lane >> 1) + 16 * i + 256 * (lane & 1))] = v[i];
        __syncwarp();
        // XL[k] = (Z[k] + conj Z[N-k]) / 2, XR[k] = (Z[k] - conj Z[N-k]) / (2i)
#pragma unroll
        for (int m = 0; m < 8; ++m) {
            const int k = lane + 32 * m;
            const float2 a = buf[nat_idx(k)];
            const float2 bb = buf[nat_idx((SSB_N_FFT - k) & (SSB_N_FFT - 1))];
            const float2 cb = make_float2(bb.x, -bb.y);
            const float2 l = add2(a, cb), r = sub2(a, cb);
            const float2 l2 = mul2(l, l), r2 = mul2(r, r);
            const float pl2 = l2.x + l2.y, pr2 = r2.x + r2.y;        // 4 |X|^2
            pbuf[k] = power == 2 ? make_float2(0.25f * pl2, 0.25f * pr2) : make_float2(0.5f * fast_sqrt(pl2), 0.5f * fast_sqrt(pr2));
        }
        if (lane == 0) {                                              // Nyquist bin: Z[256] = XL[256] + i XR[256], both real
            const float2 a = buf[nat_idx(256)];
            pbuf[256] = power == 2 ? make_float2(a.x * a.x, a.y * a.y) : make_float2(fabsf(a.x), fabsf(a.y));
        }
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float2 acc = make_float2(0.f, 0.f);
            for (int i = 0; i < row[h].y; ++i) acc = fma2(bcast(__ldg(wrow[h] + i)), pbuf[row[h].x + i], acc);
            res[h][fr] = acc;
        }
        __syncwarp();                                                 // buf / pbuf are rewritten by the next frame
#pragma unroll
        for (int q = 1; q < 10; ++q) x[q] = x[q + 5];
#pragma unroll
        for (int u = 0; u < 5; ++u) x[10 + u] = nx[u];
    }
    // out[env][j][t][ear]: 4 consecutive frames of one mel row are 32 contiguous bytes
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int j = lane + 32 * h;
        if (j >= n_mels) continue;
        float* __restrict__ o = out + (((long long)env * n_mels + j) * n_frames + t0) * 2;
#pragma unroll
        for (int fr = 0; fr < SSB_POOL; ++fr)
            if (t0 + fr < n_frames)
                *reinterpret_cast<float2*>(o + 2 * fr) = make_float2(log1pf(res[h][fr].x), log1pf(res[h][fr].y));
    }
}

// ---------------------------------------------------------------------------
// ambisonic -> binaural decode (SURVEY A11; reference: scripts/ambisonic_to_binaural.py:14-19 driving the
// closed AmbisonicBinauralizer): out[n][ear] = sum_k sum_tau (R(az) a)_k[n - 128 - tau] h[k][ear][tau].
// The rotation is folded into per-env filters g[k][tau] = sum_j R[j][k] h[j][.][tau] (sh_filters_kernel),
// then a direct-form FIR (9 channels x 256 taps, both ears as one float2) produces the (L, 2) RIR in the
// interleaved layout the convolution kernels read.
// ---------------------------------------------------------------------------
constexpr int SH_CH = 9, SH_TAPS = 256, SH_DELAY = 128;
constexpr int SH_THREADS = 128, SH_PER_THREAD = 8, SH_TILE = SH_THREADS * SH_PER_THREAD;   // outputs per CTA

// grid (filter sets); block 256: g[set][k][tau] (float2 = L,R) for set's azimuth az_deg[set], K in {1, 4, 9, 16}
template <int K>
__global__ void __launch_bounds__(SH_TAPS)
sh_filters_kernel(const float* __restrict__ hbank, const float* __restrict__ az_deg, float2* __restrict__ g) {
    const int env = blockIdx.x, tau = threadIdx.x;
    // fmodf is exact, so 2 al and 3 al keep full precision at any finite azimuth (NaN and +-inf give NaN filters)
    const float al = fmodf(az_deg[env], 360.f) * 0.017453292519943295f;
    float c1, s1, c2, s2, c3, s3;
    sincosf(al, &s1, &c1);
    sincosf(2.f * al, &s2, &c2);
    if constexpr (K == 16) sincosf(3.f * al, &s3, &c3);
    float2 h[K];
#pragma unroll
    for (int j = 0; j < K; ++j)
        h[j] = make_float2(__ldg(hbank + (j * 2 + 0) * SH_TAPS + tau), __ldg(hbank + (j * 2 + 1) * SH_TAPS + tau));
    // (R a)_j = sum_k R[j][k] a_k  =>  g_k = sum_j R[j][k] h_j; pairs (neg, pos, m): (1,3,1), (5,7,1), (4,8,2), and at
    // third order (11,13,1), (10,14,2), (9,15,3).  R[pos][pos] = c, R[pos][neg] = -s, R[neg][pos] = s, R[neg][neg] = c;
    // the m = 0 channels 0, 2, 6, 12 do not rotate.
    float2 o[K];
    o[0] = h[0];
    auto mix = [&](int neg, int pos, float c, float s) {
        o[neg] = make_float2(c * h[neg].x - s * h[pos].x, c * h[neg].y - s * h[pos].y);     // column neg: R[neg][neg] h_neg + R[pos][neg] h_pos
        o[pos] = make_float2(s * h[neg].x + c * h[pos].x, s * h[neg].y + c * h[pos].y);     // column pos: R[neg][pos] h_neg + R[pos][pos] h_pos
    };
    if constexpr (K >= 4) {
        o[2] = h[2];
        mix(1, 3, c1, s1);
    }
    if constexpr (K >= 9) {
        o[6] = h[6];
        mix(5, 7, c1, s1);
        mix(4, 8, c2, s2);
    }
    if constexpr (K == 16) {
        o[12] = h[12];
        mix(11, 13, c1, s1);
        mix(10, 14, c2, s2);
        mix(9, 15, c3, s3);
    }
#pragma unroll
    for (int k = 0; k < K; ++k) g[((long long)env * K + k) * SH_TAPS + tau] = o[k];
}

// grid (ceil(L / SH_TILE), B); block SH_THREADS.  amb[env][L][9] f32 -> out[env][L][2]
__global__ void __launch_bounds__(SH_THREADS)
sh_decode_kernel(const float* __restrict__ amb, int L, const float2* __restrict__ g, float* __restrict__ out) {
    extern __shared__ float sh_smem[];
    constexpr int SPAN = SH_TILE + SH_DELAY + SH_TAPS - 1;      // input samples feeding one tile
    float* sa = sh_smem;                                          // [9][SPAN]
    float2* sg = reinterpret_cast<float2*>(sh_smem + SH_CH * SPAN + (SH_CH * SPAN & 1));   // [9][256]
    const int env = blockIdx.y;
    const int n0 = blockIdx.x * SH_TILE;
    const int first = n0 - SH_DELAY - (SH_TAPS - 1);              // input index of sa[.][0]
    const float* __restrict__ a = amb + (long long)env * L * SH_CH;
    for (int i = threadIdx.x; i < SPAN * SH_CH; i += SH_THREADS) {
        const int pos = i / SH_CH, k = i - pos * SH_CH;            // coalesced over the interleaved (L, 9) input
        const int n = first + pos;
        sa[k * SPAN + pos] = (n >= 0 && n < L) ? __ldg(a + (long long)n * SH_CH + k) : 0.f;
    }
    for (int i = threadIdx.x; i < SH_CH * SH_TAPS; i += SH_THREADS) sg[i] = __ldg(g + (long long)env * SH_CH * SH_TAPS + i);
    __syncthreads();
    float2 acc[SH_PER_THREAD];
#pragma unroll
    for (int j = 0; j < SH_PER_THREAD; ++j) acc[j] = make_float2(0.f, 0.f);
    // thread t owns outputs n0 + t + j*SH_THREADS (j < 8): out[n] = sum_k sum_tau a_k[n - 128 - tau] g_k[tau];
    // in tile coordinates a_k[n - 128 - tau] = sa[k][(n - n0) + 255 - tau]
    for (int k = 0; k < SH_CH; ++k) {
        const float* __restrict__ ak = sa + k * SPAN + threadIdx.x + (SH_TAPS - 1);
        const float2* __restrict__ gk = sg + k * SH_TAPS;
#pragma unroll 4
        for (int tau = 0; tau < SH_TAPS; ++tau) {
            const float2 w = gk[tau];                             // broadcast
#pragma unroll
            for (int j = 0; j < SH_PER_THREAD; ++j) {
                const float x = ak[j * SH_THREADS - tau];         // conflict-free: consecutive lanes
                acc[j].x = fmaf(x, w.x, acc[j].x);
                acc[j].y = fmaf(x, w.y, acc[j].y);
            }
        }
    }
    float2* __restrict__ o = reinterpret_cast<float2*>(out) + (long long)env * L;
#pragma unroll
    for (int j = 0; j < SH_PER_THREAD; ++j) {
        const int n = n0 + threadIdx.x + j * SH_THREADS;
        if (n < L) o[n] = acc[j];
    }
}

// FFT version of the same decode (default for long responses): overlap-save with N = 4096 blocks.  The filters are
// 384 taps long including their 128-sample delay, so a block yields N - 384 = 3712 valid outputs (91 % efficient,
// against 50 % for the uniformly partitioned RIR convolution).  Per block: 9 forward transforms of the (real)
// ambisonic channels, multiply-accumulate with the 9 filter spectra G_k = FFT(delayed g_k) (both ears packed:
// real input x complex filter = left + i right), one inverse transform.  7x fewer flops than the direct form.
constexpr int SHF_LOG2N = 12;
constexpr int SHF_F = SH_DELAY + SH_TAPS;                          // 384
constexpr int SHF_HOP = (1 << SHF_LOG2N) - SHF_F;                  // 3712
// both entries refuse L > SSB_SH_MAX_L, so the grids' ceil(L / tile) and the direct form's n0 + 1023 stay inside int
static_assert((long long)SSB_SH_MAX_L + SHF_HOP - 1 <= 2147483647LL && (long long)SSB_SH_MAX_L + SH_TILE - 1 <= 2147483647LL,
              "SSB_SH_MAX_L");

// grid (K, filter sets); block 256: G[set][k][slot]
template <int K>
__global__ void __launch_bounds__(FftPlan<SHF_LOG2N>::T)
sh_filter_fft_kernel(const float2* __restrict__ g, float2* __restrict__ G, const float2* __restrict__ tw) {
    using P = FftPlan<SHF_LOG2N>;
    extern __shared__ float2 smem[];
    float2* stw = smem + P::SMEM_ELEMS;
    const int k = blockIdx.x, env = blockIdx.y, t = threadIdx.x;
    const Tw6 w0 = load_tw6<true>(tw, P::T, t);
    stage_small_twiddles<SHF_LOG2N>(stw, tw, t);
    const float2* __restrict__ gk = g + ((long long)env * K + k) * SH_TAPS;
    float2 v[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) {
        const int n = t + q * P::T;
        v[q] = (n >= SH_DELAY && n < SHF_F) ? __ldg(gk + n - SH_DELAY) : make_float2(0.f, 0.f);
    }
    fft_forward<SHF_LOG2N>(v, t, smem, w0, stw);
    store_slots<SHF_LOG2N>(G + ((long long)env * K + k) * P::N, v, t);
}

// grid (ceil(L / SHF_HOP), B); block 256
__global__ void __launch_bounds__(FftPlan<SHF_LOG2N>::T, 2)
sh_ols_kernel(const float* __restrict__ amb, int L, const float2* __restrict__ G, float* __restrict__ out,
              const float2* __restrict__ tw) {
    using P = FftPlan<SHF_LOG2N>;
    extern __shared__ float2 smem[];
    float2* stw = smem + P::SMEM_ELEMS;
    const int b = blockIdx.x, env = blockIdx.y, t = threadIdx.x;
    const Tw6 w0 = load_tw6<true>(tw, P::T, t);
    stage_small_twiddles<SHF_LOG2N>(stw, tw, t);
    const long long base = (long long)b * SHF_HOP - SHF_F;          // first input sample of this block's window
    const float* __restrict__ a = amb + (long long)env * L * SH_CH;
    const float2* __restrict__ Ge = G + (long long)env * SH_CH * P::N + t;
    float2 acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = make_float2(0.f, 0.f);
    for (int k = 0; k < SH_CH; ++k) {
        float2 v[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) {
            const long long n = base + t + q * P::T;
            v[q] = make_float2((n >= 0 && n < L) ? __ldg(a + n * SH_CH + k) : 0.f, 0.f);
        }
        if (k > 0) __syncthreads();                                 // the exchange buffer is reused by the next transform
        fft_forward<SHF_LOG2N>(v, t, smem, w0, stw);
        const float2* __restrict__ gk = Ge + (long long)k * P::N;
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[i] = cfma(v[i], __ldg(gk + i * P::T), acc[i]);
    }
    __syncthreads();
    fft_inverse<SHF_LOG2N>(acc, t, smem, tw, stw);
    constexpr float scale = 1.0f / (float)P::N;
    float2* __restrict__ o = reinterpret_cast<float2*>(out) + (long long)env * L;
#pragma unroll
    for (int q = 0; q < 16; ++q) {
        const int nl = t + q * P::T;                                // valid outputs: nl >= 384
        const long long n = (long long)b * SHF_HOP + nl - SHF_F;
        if (nl >= SHF_F && n < L) o[n] = make_float2(acc[q].x * scale, acc[q].y * scale);
    }
}

// Several azimuths per input (ssb_sh_decode_multi_batch): output b = in * n_az + a decodes input `in` with filter set
// a.  Both forms read each input once per CTA and reuse it for every azimuth.  Each output's arithmetic is the same
// sequence whatever n_az is, so a row of an n_az = 4 decode is bit-identical to the n_az = 1 decode at its azimuth.

// grid (ceil(L / SH_TILE), n_inputs); block SH_THREADS.  amb[in][L][K] -> out[in][a][L][2].  The input tile is staged
// once; the filter sets are staged one after the other against it (four K = 16 sets would not fit beside the tile).
template <int K>
__global__ void __launch_bounds__(SH_THREADS)
sh_decode_multi_kernel(const float* __restrict__ amb, int L, int n_az, const float2* __restrict__ g, float* __restrict__ out) {
    extern __shared__ float sh_smem[];
    constexpr int SPAN = SH_TILE + SH_DELAY + SH_TAPS - 1;
    float* sa = sh_smem;                                          // [K][SPAN]
    float2* sg = reinterpret_cast<float2*>(sh_smem + K * SPAN + (K * SPAN & 1));   // [K][256]
    const int in = blockIdx.y;
    const int n0 = blockIdx.x * SH_TILE;
    const int first = n0 - SH_DELAY - (SH_TAPS - 1);
    const float* __restrict__ a = amb + (long long)in * L * K;
    for (int i = threadIdx.x; i < SPAN * K; i += SH_THREADS) {
        const int pos = i / K, k = i - pos * K;
        const int n = first + pos;
        sa[k * SPAN + pos] = (n >= 0 && n < L) ? __ldg(a + (long long)n * K + k) : 0.f;
    }
    for (int az = 0; az < n_az; ++az) {
        if (az > 0) __syncthreads();                              // every thread is done with the previous set
        for (int i = threadIdx.x; i < K * SH_TAPS; i += SH_THREADS) sg[i] = __ldg(g + (long long)az * K * SH_TAPS + i);
        __syncthreads();
        float2 acc[SH_PER_THREAD];
#pragma unroll
        for (int j = 0; j < SH_PER_THREAD; ++j) acc[j] = make_float2(0.f, 0.f);
        for (int k = 0; k < K; ++k) {
            const float* __restrict__ ak = sa + k * SPAN + threadIdx.x + (SH_TAPS - 1);
            const float2* __restrict__ gk = sg + k * SH_TAPS;
#pragma unroll 4
            for (int tau = 0; tau < SH_TAPS; ++tau) {
                const float2 w = gk[tau];
#pragma unroll
                for (int j = 0; j < SH_PER_THREAD; ++j) {
                    const float x = ak[j * SH_THREADS - tau];
                    acc[j].x = fmaf(x, w.x, acc[j].x);
                    acc[j].y = fmaf(x, w.y, acc[j].y);
                }
            }
        }
        float2* __restrict__ o = reinterpret_cast<float2*>(out) + ((long long)in * n_az + az) * L;
#pragma unroll
        for (int j = 0; j < SH_PER_THREAD; ++j) {
            const int n = n0 + threadIdx.x + j * SH_THREADS;
            if (n < L) o[n] = acc[j];
        }
    }
}

// grid (ceil(L / SHF_HOP), n_inputs); block 256.  Each window's K channels are forward-transformed once per group of
// AC azimuths and multiply-accumulated into AC register accumulators, one inverse transform each: K + AC transforms
// per group instead of AC * (K + 1).
template <int K, int AC>
__global__ void __launch_bounds__(FftPlan<SHF_LOG2N>::T, AC == 1 ? 2 : 1)
sh_ols_multi_kernel(const float* __restrict__ amb, int L, int n_az, const float2* __restrict__ G, float* __restrict__ out,
                    const float2* __restrict__ tw) {
    using P = FftPlan<SHF_LOG2N>;
    extern __shared__ float2 smem[];
    float2* stw = smem + P::SMEM_ELEMS;
    const int b = blockIdx.x, in = blockIdx.y, t = threadIdx.x;
    const Tw6 w0 = load_tw6<true>(tw, P::T, t);
    stage_small_twiddles<SHF_LOG2N>(stw, tw, t);
    const long long base = (long long)b * SHF_HOP - SHF_F;
    const float* __restrict__ a = amb + (long long)in * L * K;
    for (int a0 = 0; a0 < n_az; a0 += AC) {
        float2 acc[AC][16];
#pragma unroll
        for (int c = 0; c < AC; ++c)
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[c][i] = make_float2(0.f, 0.f);
        for (int k = 0; k < K; ++k) {
            float2 v[16];
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const long long n = base + t + q * P::T;
                v[q] = make_float2((n >= 0 && n < L) ? __ldg(a + n * K + k) : 0.f, 0.f);
            }
            if (k > 0 || a0 > 0) __syncthreads();                   // the exchange buffer is reused by this transform
            fft_forward<SHF_LOG2N>(v, t, smem, w0, stw);
#pragma unroll
            for (int c = 0; c < AC; ++c) {
                if (a0 + c >= n_az) break;
                const float2* __restrict__ gk = G + ((long long)(a0 + c) * K + k) * P::N + t;
#pragma unroll
                for (int i = 0; i < 16; ++i) acc[c][i] = cfma(v[i], __ldg(gk + i * P::T), acc[c][i]);
            }
        }
#pragma unroll
        for (int c = 0; c < AC; ++c) {
            if (a0 + c >= n_az) break;
            __syncthreads();
            fft_inverse<SHF_LOG2N>(acc[c], t, smem, tw, stw);
            constexpr float scale = 1.0f / (float)P::N;
            float2* __restrict__ o = reinterpret_cast<float2*>(out) + ((long long)in * n_az + a0 + c) * L;
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const int nl = t + q * P::T;
                const long long n = (long long)b * SHF_HOP + nl - SHF_F;
                if (nl >= SHF_F && n < L) o[n] = make_float2(acc[c][q].x * scale, acc[c][q].y * scale);
            }
        }
    }
}

// ---------------------------------------------------------------------------
// small kernels
// ---------------------------------------------------------------------------
__global__ void crossfade_kernel(const float* __restrict__ prev, float* __restrict__ cur, int n_fade,
                                 long long wave_stride, const uint8_t* __restrict__ enable) {
    const int row = blockIdx.y;                  // env*2 + ear
    if (enable && !enable[row >> 1]) return;
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m > n_fade) return;
    // continuous_simulator.py:48-51: x2_weight = arange(n+1)/n ; x1_weight = flip(x2_weight)
    const float w2 = (float)m / (float)n_fade;
    const float w1 = (float)(n_fade - m) / (float)n_fade;
    const long long o = (long long)row * wave_stride + m;
    cur[o] = prev[o] * w1 + cur[o] * w2;
}

// Intensity sensor of AV-WaN (ss_baselines/av_wan/avwan_sensors.py:91-100): onset = the first sample (min
// over ears) exceeding 10 % of the clip maximum; result = mean square of the num_frame samples after it.
// grid (B); block 256
__global__ void __launch_bounds__(256)
intensity_kernel(const float* __restrict__ wave, long long wave_stride, int sr, int num_frame, float* __restrict__ out) {
    __shared__ float sf[256];
    __shared__ int si[256];
    const int env = blockIdx.x, t = threadIdx.x;
    const float* __restrict__ yl = wave + (long long)env * 2 * wave_stride;
    const float* __restrict__ yr = yl + wave_stride;
    float m = -INFINITY;
    for (int n = t; n < sr; n += 256) m = fmaxf(m, fmaxf(yl[n], yr[n]));
    sf[t] = m;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) { if (t < s) sf[t] = fmaxf(sf[t], sf[t + s]); __syncthreads(); }
    const float thr = 0.1f * sf[0];
    __syncthreads();
    // first index per ear with value > thr (np.argmax of an all-False row is 0), then min over ears
    int fl = sr, fr = sr;
    for (int n = t; n < sr; n += 256) {
        if (yl[n] > thr && n < fl) fl = n;
        if (yr[n] > thr && n < fr) fr = n;
    }
    si[t] = fl;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) { if (t < s) si[t] = min(si[t], si[t + s]); __syncthreads(); }
    const int first_l = si[0] == sr ? 0 : si[0];
    __syncthreads();
    si[t] = fr;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) { if (t < s) si[t] = min(si[t], si[t + s]); __syncthreads(); }
    const int first_r = si[0] == sr ? 0 : si[0];
    const int idx = min(first_l, first_r);
    const int end = min(idx + num_frame, sr);               // numpy slicing clips at the end of the clip
    float acc = 0.f;
    for (int n = idx + t; n < end; n += 256) acc += yl[n] * yl[n] + yr[n] * yr[n];
    __syncthreads();
    sf[t] = acc;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) { if (t < s) sf[t] += sf[t + s]; __syncthreads(); }
    if (t == 0) out[env] = end > idx ? sf[0] / (float)(2 * (end - idx)) : nanf("");
}

// ---------------------------------------------------------------------------
// SURVEY.md N2: the first layer of the policy's audio encoder fused with the layout change.  AudioCNN.forward
// (ss_baselines/av_nav/models/audio_cnn.py:79-89) permutes the (N, 65, T', 2) observation to (N, 2, 65, T') and runs
// Conv2d(2 -> 32, 8x8 / 4, or 5x5 / 2 for inputs under 30 pixels) + ReLU; here the convolution reads the observation
// in the layout the spectrogram kernel wrote it (ears interleaved) and writes (N, OC, H1, W1): no permuted copy, one
// launch.  Inference only (rollout collection runs under no_grad, ppo_trainer.py:131-146); the PPO update keeps
// PyTorch's layer.  grid (H1, N); block (W1 * OC) <= 1024; dynamic smem: KH input rows + all weights.
// ---------------------------------------------------------------------------

// One output of the first layer: acc + sum over (kh, kw) of left * w0 + right * w1, in this order.  r points at input
// pixel (oh * SH, ow * SW) of an ears-interleaved [rows][W][2] tile (row stride 2 W floats); w0 / w1 are the
// [KH][KW] filters of the output channel for channel 0 (left ear) and channel 1 (right ear).
__device__ __forceinline__ float conv1_point(const float* __restrict__ r, int W, const float* __restrict__ w0,
                                             const float* __restrict__ w1, int KH, int KW, float acc) {
    for (int kh = 0; kh < KH; ++kh, r += 2 * W) {
        for (int kw = 0; kw < KW; ++kw) {
            acc = fmaf(r[2 * kw], w0[kh * KW + kw], acc);           // channel 0 = left ear
            acc = fmaf(r[2 * kw + 1], w1[kh * KW + kw], acc);       // channel 1 = right ear
        }
    }
    return acc;
}

// torch's ReLU: NaN stays NaN (fmaxf(NaN, 0) would return 0 and hide it from the caller)
__device__ __forceinline__ float relu_keep_nan(float v) { return v > 0.f || v != v ? v : 0.f; }

__global__ void audio_conv1_kernel(const float* __restrict__ spec, int H, int W, const float* __restrict__ weight,
                                   const float* __restrict__ bias, int OC, int KH, int KW, int SH, int SW, int H1, int W1,
                                   int relu, float* __restrict__ out) {
    extern __shared__ float c1_smem[];
    float* rows = c1_smem;                                  // [KH][W][2]
    float* wsm = c1_smem + KH * W * 2;                      // [OC][2][KH][KW]
    const int oh = blockIdx.x, n = blockIdx.y, tid = threadIdx.x;
    const float* __restrict__ in = spec + ((long long)n * H + (long long)oh * SH) * W * 2;
    for (int i = tid; i < KH * W * 2; i += blockDim.x) rows[i] = __ldg(in + i);
    for (int i = tid; i < OC * 2 * KH * KW; i += blockDim.x) wsm[i] = __ldg(weight + i);
    __syncthreads();
    const int ow = tid % W1, oc = tid / W1;
    if (oc >= OC) return;
    float acc = bias ? __ldg(bias + oc) : 0.f;
    acc = conv1_point(rows + ow * SW * 2, W, wsm + (oc * 2 + 0) * KH * KW, wsm + (oc * 2 + 1) * KH * KW, KH, KW, acc);
    if (relu) acc = relu_keep_nan(acc);
    out[(((long long)n * OC + oc) * H1 + oh) * W1 + ow] = acc;
}

// ---------------------------------------------------------------------------
// The whole AudioCNN.cnn at rollout time (ss_baselines/{av_nav,av_wan,savi}/models/audio_cnn.py: Conv2d(2 -> C1) ReLU
// Conv2d(C1 -> C2) ReLU Conv2d(C2 -> C3) Flatten Linear ReLU) in two launches:
//  - audio_encoder_conv_kernel: conv1 (+ReLU) -> conv2 (+ReLU) -> conv3 for one env per cluster of ENC_CL CTAs.  Every
//    CTA stages the env's observation and keeps the FULL conv1 and conv2 activations in its shared memory; it computes
//    a contiguous slice of each layer's output channels and stores every value into all ENC_CL CTAs' copies over
//    distributed shared memory, with a cluster barrier between layers, so each layer's inner loop reads local shared
//    memory only.  Before each layer the CTA copies its slice of that layer's weights (contiguous in torch's
//    [OC][IC][KH][KW]) into shared memory with one coalesced pass: read in the inner loop, every weight would otherwise
//    be a dependent L2 round trip shared by the few warps of the CTA.  conv3 goes straight to the (B, F) features in
//    torch's Flatten order (c, h, w).
//  - audio_encoder_linear_kernel: out[n][j] = act(b[j] + sum_f W[j][f] x[n][f]).  A CTA owns LIN_ROWS output rows for
//    a tile of LIN_ENVS envs, so each tile of envs streams the weight once; its LIN_WARPS warps split the features and
//    their partial sums are added in warp order.
// Every output is a fixed sequence of fmaf (over (ic, kh, kw), or over f per lane followed by a fixed reduction tree), so
// an env's results are bit-identical whatever the batch size and its position in the batch.  conv1 is conv1_point, the
// same arithmetic as audio_conv1_kernel.  SAVi with a distractor sound (savi/models/audio_cnn.py:135-150) concatenates
// the env's category row, broadcast over H x W, after the two ears: conv1 then has 2 + n_labels input channels, and the
// label channels enter as a per-(env, channel) bias folded in shared memory (no extra launch, no extra shared memory).
// ---------------------------------------------------------------------------
constexpr int ENC_CL = 8;                 // CTAs per env: 16 envs fill 128 of the 132 SMs
constexpr int ENC_TPB = 256;
constexpr int ENC_OCT = 2;                // conv2 / conv3: output channels per thread (register tile)
constexpr int ENC_SMEM_MAX = 227 * 1024;  // the per-CTA opt-in limit of sm_90

struct EncLayer { const float* w; const float* b; int oc, kh, kw, sh, sw, relu, ho, wo; };
// labels: [B][label_stride] floats, columns 0..n_labels-1 are conv1's input channels 2..n_labels+1 (SAVi's category)
struct EncParams { EncLayer l[3]; int H, W; const float* labels; long long label_stride; int n_labels; };

// output channels per cluster rank, and the weight floats a rank stages for a layer with IC inputs and KK taps
__host__ __device__ __forceinline__ int enc_chunk(int OC) { return (OC + ENC_CL - 1) / ENC_CL; }
__host__ __device__ __forceinline__ long long enc_wslice(int OC, long long IC, int KK) { return (long long)enc_chunk(OC) * IC * KK; }

// channels [c0, c1) of a layer with OC outputs computed by cluster rank `rank`
__device__ __forceinline__ void enc_slice(int OC, int rank, int& c0, int& c1) {
    c0 = min(OC, rank * enc_chunk(OC));
    c1 = min(OC, c0 + enc_chunk(OC));
}

// copy this rank's weight slice (channels [c0, c1), per = IC KK floats each) into shared memory
__device__ __forceinline__ void enc_stage_weights(float* __restrict__ ws, const float* __restrict__ w, int c0, int c1, int per) {
    const float* __restrict__ src = w + (long long)c0 * per;
    const int n = (c1 - c0) * per;
#pragma unroll 4
    for (int i = threadIdx.x; i < n; i += ENC_TPB) ws[i] = __ldg(src + i);
}

// conv2 / conv3 over a channels-first [IC][Hi][Wi] activation in local shared memory: this rank's channel slice, ENC_OCT
// channels per thread at one output pixel, weights from the staged slice ws.  dst == nullptr: store into every cluster
// CTA's copy of the [OC][Ho][Wo] buffer at offset `dst_smem`; otherwise store to global memory at dst.  KH_, KW_ > 0
// fix the kernel size at compile time (the reference's 3x3 and 4x4 layers: the tap loops unroll, so the shared-memory
// loads of a tap row issue together); 0 reads it from L.  The arithmetic is the same either way.
template <int KH_, int KW_>
__device__ __forceinline__ void enc_conv_chw(cg::cluster_group& cluster, int rank, const float* __restrict__ in, int IC,
                                            int Hi, int Wi, const EncLayer& L, const float* __restrict__ ws,
                                            float* dst_smem, float* __restrict__ dst) {
    int c0, c1;
    enc_slice(L.oc, rank, c0, c1);
    const int KH = KH_ > 0 ? KH_ : L.kh, KW = KW_ > 0 ? KW_ : L.kw;
    const int HWo = L.ho * L.wo, KK = KH * KW, wstride = IC * KK;
    const int groups = (c1 - c0 + ENC_OCT - 1) / ENC_OCT;
    for (int idx = threadIdx.x; idx < groups * HWo; idx += ENC_TPB) {
        const int g = idx / HWo, pos = idx % HWo;
        const int oc0 = c0 + g * ENC_OCT, oh = pos / L.wo, ow = pos % L.wo;
        const int nvalid = min(ENC_OCT, c1 - oc0);
        const float* __restrict__ wp[ENC_OCT];
        float acc[ENC_OCT];
#pragma unroll
        for (int t = 0; t < ENC_OCT; ++t) {
            const int oc = oc0 + min(t, nvalid - 1);          // the tail of a slice recomputes its last channel
            wp[t] = ws + (oc - c0) * wstride;
            acc[t] = L.b ? __ldg(L.b + oc) : 0.f;
        }
        const float* __restrict__ x0 = in + oh * L.sh * Wi + ow * L.sw;
        for (int ic = 0; ic < IC; ++ic) {
            const float* __restrict__ x1 = x0 + ic * Hi * Wi;
            const int wofs = ic * KK;
#pragma unroll
            for (int kh = 0; kh < KH; ++kh) {
#pragma unroll
                for (int kw = 0; kw < KW; ++kw) {
                    const float x = x1[kh * Wi + kw];
#pragma unroll
                    for (int t = 0; t < ENC_OCT; ++t) acc[t] = fmaf(x, wp[t][wofs + kh * KW + kw], acc[t]);
                }
            }
        }
#pragma unroll
        for (int t = 0; t < ENC_OCT; ++t) {
            if (t >= nvalid) break;
            const float v = L.relu ? relu_keep_nan(acc[t]) : acc[t];
            const int o = (oc0 + t) * HWo + pos;
            if (dst) {
                dst[o] = v;
            } else {
#pragma unroll
                for (int r = 0; r < ENC_CL; ++r) *cluster.map_shared_rank(dst_smem + o, r) = v;
            }
        }
    }
}

__device__ __forceinline__ void enc_conv_layer(cg::cluster_group& cluster, int rank, const float* __restrict__ in, int IC,
                                              int Hi, int Wi, const EncLayer& L, const float* __restrict__ ws,
                                              float* dst_smem, float* __restrict__ dst) {
    if (L.kh == 3 && L.kw == 3)
        enc_conv_chw<3, 3>(cluster, rank, in, IC, Hi, Wi, L, ws, dst_smem, dst);
    else if (L.kh == 4 && L.kw == 4)
        enc_conv_chw<4, 4>(cluster, rank, in, IC, Hi, Wi, L, ws, dst_smem, dst);
    else
        enc_conv_chw<0, 0>(cluster, rank, in, IC, Hi, Wi, L, ws, dst_smem, dst);
}

// A label channel is constant over H x W and conv1 is unpadded, so it adds sum_c l[c] sum_k W[oc][2 + c][k] to every
// output of channel oc: fold that into the bias, in the staged conv1 slice ws ([c1 - c0][2 + NL][KK] floats).  First
// the tap sum of each (channel, label) in k order, stored over its first tap; then per channel b[oc] + the label terms
// in c order, stored over the first tap of label 0.  Each value is overwritten only by the thread that read it; the ear
// taps stay as staged.
__device__ __forceinline__ void enc_fold_label_bias(float* ws, const float* __restrict__ bias, const float* __restrict__ lab,
                                                    int NL, int KK, int c0, int c1) {
    const int per = (2 + NL) * KK;
    __syncthreads();                                         // the slice is staged
    for (int idx = threadIdx.x; idx < (c1 - c0) * NL; idx += ENC_TPB) {
        float* t = ws + (idx / NL) * per + (2 + idx % NL) * KK;
        float s = t[0];
        for (int k = 1; k < KK; ++k) s += t[k];
        t[0] = s;
    }
    __syncthreads();
    for (int ch = threadIdx.x; ch < c1 - c0; ch += ENC_TPB) {
        float* t = ws + ch * per + 2 * KK;
        float acc = bias ? __ldg(bias + c0 + ch) : 0.f;
        for (int c = 0; c < NL; ++c) acc = fmaf(__ldg(lab + c), t[c * KK], acc);
        t[0] = acc;
    }
}

// grid (ENC_CL, B), cluster (ENC_CL, 1, 1), block ENC_TPB; dynamic smem (H W 2 + C1 H1 W1 + C2 H2 W2 + the largest
// weight slice) floats.  LABELS: SAVi with a distractor sound, p.n_labels > 0 category channels; without, the labels
// are unused and the code is the ears-only encoder's exactly
template <bool LABELS>
__global__ void __cluster_dims__(ENC_CL, 1, 1) __launch_bounds__(ENC_TPB)
audio_encoder_conv_kernel(const float* __restrict__ spec, const EncParams p, float* __restrict__ feat) {
    extern __shared__ float enc_smem[];
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = (int)cluster.block_rank(), n = blockIdx.y, tid = threadIdx.x;
    const EncLayer &L1 = p.l[0], &L2 = p.l[1], &L3 = p.l[2];
    const int obs_elems = p.H * p.W * 2;
    float* obs = enc_smem;                                   // [H][W][2], as the spectrogram kernel wrote it
    float* a1 = obs + obs_elems;                             // [C1][H1][W1]
    float* a2 = a1 + L1.oc * L1.ho * L1.wo;                  // [C2][H2][W2]
    float* ws = a2 + L2.oc * L2.ho * L2.wo;                  // this rank's weight slice of the current layer
    const float* __restrict__ src = spec + (long long)n * obs_elems;
    const int KK1 = L1.kh * L1.kw, NL = LABELS ? p.n_labels : 0, WS1 = (2 + NL) * KK1;   // conv1 floats per channel
    int c0, c1;
    enc_slice(L1.oc, rank, c0, c1);
    for (int i = tid; i < obs_elems; i += ENC_TPB) obs[i] = __ldg(src + i);
    enc_stage_weights(ws, L1.w, c0, c1, WS1);
    if (LABELS) enc_fold_label_bias(ws, L1.b, p.labels + n * p.label_stride, NL, KK1, c0, c1);
    cluster.sync();                                          // observation and weights staged, every peer is running
    {
        const int HW1 = L1.ho * L1.wo;
        for (int idx = tid; idx < (c1 - c0) * HW1; idx += ENC_TPB) {
            const int oc = c0 + idx / HW1, pos = idx % HW1;
            const int oh = pos / L1.wo, ow = pos % L1.wo;
            const float* w = ws + (oc - c0) * WS1;
            float acc = LABELS ? w[2 * KK1] : L1.b ? __ldg(L1.b + oc) : 0.f;
            acc = conv1_point(obs + (oh * L1.sh * p.W + ow * L1.sw) * 2, p.W, w, w + KK1, L1.kh, L1.kw, acc);
            if (L1.relu) acc = relu_keep_nan(acc);
#pragma unroll
            for (int r = 0; r < ENC_CL; ++r) *cluster.map_shared_rank(a1 + oc * HW1 + pos, r) = acc;
        }
    }
    __syncthreads();                                         // this CTA is done with the conv1 weights
    enc_slice(L2.oc, rank, c0, c1);
    enc_stage_weights(ws, L2.w, c0, c1, L1.oc * L2.kh * L2.kw);
    cluster.sync();                                          // every copy of a1 is complete
    enc_conv_layer(cluster, rank, a1, L1.oc, L1.ho, L1.wo, L2, ws, a2, nullptr);
    __syncthreads();
    enc_slice(L3.oc, rank, c0, c1);
    enc_stage_weights(ws, L3.w, c0, c1, L2.oc * L3.kh * L3.kw);
    cluster.sync();                                          // every copy of a2 is complete; no DSMEM access after this
    const long long F = (long long)L3.oc * L3.ho * L3.wo;
    enc_conv_layer(cluster, rank, a2, L2.oc, L2.ho, L2.wo, L3, ws, nullptr, feat + n * F);
}

constexpr int LIN_ENVS = 16;              // envs per tile (the rollout batch of one GPU)
constexpr int LIN_ROWS = 4;               // output rows per CTA: each loaded x value feeds LIN_ROWS FMAs
constexpr int LIN_WARPS = 8;              // warps splitting the features

// grid (ceil(hidden / LIN_ROWS), ceil(B / LIN_ENVS)), block 32 LIN_WARPS.  Lane l of warp w sums the features
// f = l + 32 (w + LIN_WARPS k) in increasing k; the lanes are combined by a butterfly, the warps in warp order.
__global__ void __launch_bounds__(32 * LIN_WARPS)
audio_encoder_linear_kernel(const float* __restrict__ x, int B, int F, const float* __restrict__ weight,
                            const float* __restrict__ bias, int hidden, int relu, float* __restrict__ out) {
    __shared__ float red[LIN_WARPS][LIN_ROWS * LIN_ENVS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j0 = blockIdx.x * LIN_ROWS, e0 = blockIdx.y * LIN_ENVS;
    const int ne = min(LIN_ENVS, B - e0);
    const float* __restrict__ wr[LIN_ROWS];
#pragma unroll
    for (int r = 0; r < LIN_ROWS; ++r) wr[r] = weight + (long long)min(j0 + r, hidden - 1) * F;   // rows past hidden: not stored
    const float* __restrict__ xe = x + (long long)e0 * F;
    float acc[LIN_ROWS][LIN_ENVS];
#pragma unroll
    for (int r = 0; r < LIN_ROWS; ++r)
#pragma unroll
        for (int e = 0; e < LIN_ENVS; ++e) acc[r][e] = 0.f;
    for (int f = warp * 32 + lane; f < F; f += 32 * LIN_WARPS) {
        float w[LIN_ROWS];
#pragma unroll
        for (int r = 0; r < LIN_ROWS; ++r) w[r] = __ldg(wr[r] + f);
#pragma unroll
        for (int e = 0; e < LIN_ENVS; ++e) {
            const float xv = __ldg(xe + (long long)min(e, ne - 1) * F + f);   // envs past B: not stored
#pragma unroll
            for (int r = 0; r < LIN_ROWS; ++r) acc[r][e] = fmaf(w[r], xv, acc[r][e]);
        }
    }
    // butterfly sum over the lanes: every lane ends with the same total (a + b == b + a), in a fixed order
#pragma unroll
    for (int r = 0; r < LIN_ROWS; ++r)
#pragma unroll
        for (int e = 0; e < LIN_ENVS; ++e)
#pragma unroll
            for (int m = 16; m >= 1; m >>= 1) acc[r][e] += __shfl_xor_sync(0xffffffffu, acc[r][e], m);
#pragma unroll
    for (int r = 0; r < LIN_ROWS; ++r)
#pragma unroll
        for (int e = 0; e < LIN_ENVS; ++e)
            if (lane == ((r * LIN_ENVS + e) & 31)) red[warp][r * LIN_ENVS + e] = acc[r][e];
    __syncthreads();
    const int t = threadIdx.x, r = t / LIN_ENVS, e = t % LIN_ENVS, j = j0 + r;
    if (t < LIN_ROWS * LIN_ENVS && j < hidden && e < ne) {
        float s = red[0][t];
#pragma unroll
        for (int w = 1; w < LIN_WARPS; ++w) s += red[w][t];
        const float v = (bias ? __ldg(bias + j) : 0.f) + s;
        out[(long long)(e0 + e) * hidden + j] = relu ? relu_keep_nan(v) : v;
    }
}

// ---------------------------------------------------------------------------
// The whole VisualCNN.cnn at rollout time (ss_baselines/av_nav/models/visual_cnn.py:137-161, av_wan :95-118 and savi
// without semantic channels: permute, RGB / 255, cat(RGB, depth), Conv2d ReLU Conv2d ReLU Conv2d Flatten Linear ReLU)
// in two launches, visual_encoder_conv_kernel then audio_encoder_linear_kernel.  The 128 x 128 observation (256 KB for
// RGB-D) does not fit next to the conv1 activations (123 KB) in one CTA, so unlike audio_encoder_conv_kernel the
// observation is never staged whole: cluster rank r computes conv1 output rows r, r + ENC_CL, ... for every channel,
// staging only the KH1 input rows of one output row at a time (RGB scaled on load, channels RGB first, then depth),
// and stores each value into every CTA's copy of the conv1 activations over DSMEM.  During conv1 the region that later
// holds the conv2 activations holds the conv1 weights, transposed to [ic kh kw][oc] so that the 32 lanes of a warp
// (32 channels at the same VIS_PIX pixels) read consecutive weights and one broadcast input value per tap.  conv2 and
// conv3 are enc_conv_chw, as in the audio encoder.  conv1 sums bias, then (ic, kh, kw) in order.
// ---------------------------------------------------------------------------
constexpr int VIS_PIX = 4;                // conv1: output pixels of one row per thread (register tile)

// rgb [B][H][W][n_rgb] (scaled by 1/255 on load), depth [B][H][W][n_depth]; conv1 has n_rgb + n_depth input channels
struct VisParams { EncLayer l[3]; int H, W, n_rgb, n_depth; const float* rgb; const float* depth; };

// floats of the region after the conv1 activations: the conv2 activations, or during conv1 the transposed conv1
// weights and the staged input rows of one output row
__host__ __device__ __forceinline__ long long vis_region2(const VisParams& p) {
    const long long ic = p.n_rgb + p.n_depth;
    const long long conv1 = (long long)p.l[0].oc * ic * p.l[0].kh * p.l[0].kw + ic * p.l[0].kh * p.W;
    const long long a2 = (long long)p.l[1].oc * p.l[1].ho * p.l[1].wo;
    return a2 > conv1 ? a2 : conv1;
}

// grid (ENC_CL, B), cluster (ENC_CL, 1, 1), block ENC_TPB; dynamic smem (C1 H1 W1 + vis_region2 + the largest conv2 /
// conv3 weight slice) floats
__global__ void __cluster_dims__(ENC_CL, 1, 1) __launch_bounds__(ENC_TPB)
visual_encoder_conv_kernel(const VisParams p, float* __restrict__ feat) {
    extern __shared__ float enc_smem[];
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = (int)cluster.block_rank(), n = blockIdx.y, tid = threadIdx.x;
    const EncLayer &L1 = p.l[0], &L2 = p.l[1], &L3 = p.l[2];
    const int IC = p.n_rgb + p.n_depth, KH = L1.kh, KW = L1.kw, K1 = IC * KH * KW, C1 = L1.oc, HW1 = L1.ho * L1.wo;
    float* a1 = enc_smem;                                    // [C1][H1][W1]
    float* a2 = a1 + C1 * HW1;                               // [C2][H2][W2]
    float* ws = a2 + vis_region2(p);                         // this rank's weight slice of conv2 / conv3
    float* w1 = a2;                                          // conv1 only: [K1][C1]
    float* xs = w1 + C1 * K1;                                // conv1 only: [IC][KH][W], one output row's input rows
    for (int i = tid; i < C1 * K1; i += ENC_TPB) w1[(i % K1) * C1 + i / K1] = __ldg(L1.w + i);
    const long long pix0 = (long long)n * p.H * p.W;
    const float* __restrict__ rgb = p.rgb + pix0 * p.n_rgb;
    const float* __restrict__ depth = p.depth + pix0 * p.n_depth;
    const float inv255 = 1.0f / 255.0f;                      // torch's CUDA x / 255.0: x times the float reciprocal
    const int npg = (L1.wo + VIS_PIX - 1) / VIS_PIX;
    cluster.sync();                                          // every peer is running before any DSMEM store
    for (int oh = rank; oh < L1.ho; oh += ENC_CL) {
        __syncthreads();                                     // w1 staged; the previous row's xs is consumed
        const long long row0 = (long long)oh * L1.sh * p.W;
        for (int i = tid; i < KH * p.W * IC; i += ENC_TPB) {
            const int c = i % IC, col = (i / IC) % p.W, kh = i / (IC * p.W);
            const long long px = row0 + (long long)kh * p.W + col;
            xs[(c * KH + kh) * p.W + col] = c < p.n_rgb ? __ldg(rgb + px * p.n_rgb + c) * inv255
                                                         : __ldg(depth + px * p.n_depth + (c - p.n_rgb));
        }
        __syncthreads();
        for (int idx = tid; idx < C1 * npg; idx += ENC_TPB) {
            const int oc = idx % C1, ow0 = (idx / C1) * VIS_PIX, nvalid = min(VIS_PIX, L1.wo - ow0);
            int xo[VIS_PIX];
            float acc[VIS_PIX];
            const float b = L1.b ? __ldg(L1.b + oc) : 0.f;
#pragma unroll
            for (int t = 0; t < VIS_PIX; ++t) {
                xo[t] = (ow0 + min(t, nvalid - 1)) * L1.sw;  // the tail of a row recomputes its last pixel
                acc[t] = b;
            }
            for (int c = 0; c < IC; ++c)
                for (int kh = 0; kh < KH; ++kh) {
                    const float* __restrict__ xr = xs + (c * KH + kh) * p.W;
                    const float* __restrict__ wr = w1 + ((c * KH + kh) * KW) * C1 + oc;
                    for (int kw = 0; kw < KW; ++kw) {
                        const float w = wr[kw * C1];
#pragma unroll
                        for (int t = 0; t < VIS_PIX; ++t) acc[t] = fmaf(xr[xo[t] + kw], w, acc[t]);
                    }
                }
#pragma unroll
            for (int t = 0; t < VIS_PIX; ++t) {
                if (t >= nvalid) break;
                const float v = L1.relu ? relu_keep_nan(acc[t]) : acc[t];
                const int o = oc * HW1 + oh * L1.wo + ow0 + t;
#pragma unroll
                for (int r = 0; r < ENC_CL; ++r) *cluster.map_shared_rank(a1 + o, r) = v;
            }
        }
    }
    int c0, c1;
    enc_slice(L2.oc, rank, c0, c1);
    enc_stage_weights(ws, L2.w, c0, c1, C1 * L2.kh * L2.kw);
    cluster.sync();                                          // every copy of a1 is complete and every rank is done with w1 / xs
    enc_conv_layer(cluster, rank, a1, C1, L1.ho, L1.wo, L2, ws, a2, nullptr);
    __syncthreads();
    enc_slice(L3.oc, rank, c0, c1);
    enc_stage_weights(ws, L3.w, c0, c1, L2.oc * L3.kh * L3.kw);
    cluster.sync();                                          // every copy of a2 is complete; no DSMEM access after this
    const long long F = (long long)L3.oc * L3.ho * L3.wo;
    enc_conv_layer(cluster, rank, a2, L2.oc, L2.ho, L2.wo, L3, ws, nullptr, feat + n * F);
}

// ---------------------------------------------------------------------------
// The whole MapCNN.cnn at rollout time (ss_baselines/av_wan/models/map_cnn.py:65-104: permute, Conv2d ReLU Conv2d ReLU
// Conv2d Flatten Linear ReLU, unpadded) in two launches, map_encoder_conv_kernel then audio_encoder_linear_kernel.  The
// geometric map's conv1 activations (300 KB at MAP_SIZE 200, 780 KB at 400) do not fit one CTA, so unlike the audio and
// visual kernels no CTA holds a full copy: they are spread over the ENC_CL CTAs of the env's cluster.
//  - conv1: rank r computes output rows r, r + ENC_CL, ... for every channel from the KH1 input rows of each, staged
//    channels first (the channels-last rows are contiguous in global memory), and keeps them locally.  The conv1
//    weights are staged transposed to [ic kh kw][oc], as in visual_encoder_conv_kernel.
//  - conv2, one output row at a time: every rank gathers the KH2 conv1 rows that row reads from their owners over DSMEM,
//    then computes its enc_slice of the output channels into a local slice.
//  - conv3: after a cluster barrier every rank gathers the whole conv2 output from the ranks' slices into the region
//    conv1 used and computes its channel slice with enc_conv_chw, as the audio encoder does, straight to the features.
// Every sum is bias, then (ic, kh, kw) in order.  Shared-memory layout (floats, formula in include/ssb200.h):
//   conv1 phase  [a1: C1 ceil(H1 / ENC_CL) W1][w1: K1 C1][xs: IC KH1 W]          ... [s2]
//   conv2 phase  [a1][g2: C1 KH2 W1][ws2: ceil(C2 / ENC_CL) C1 KH2 KW2]          ... [s2: ceil(C2 / ENC_CL) H2 W2]
//   conv3 phase  [a2: C2 H2 W2][ws3: ceil(C3 / ENC_CL) C2 KH3 KW3]               ... [s2]
// s2 sits past the end of all three phases, so peers can read it while the rank fills a2.
// ---------------------------------------------------------------------------
constexpr int MAP_PIX = 4;                // conv1: output pixels of one row per thread (register tile)
constexpr int MAP_BATCH = 8;              // staging copies: loads in flight per thread before their stores

// map [B][H][W][C]; conv1 has C input channels
struct MapParams { EncLayer l[3]; int C, H, W; const float* map; };

// store(i, load(i)) for i in [0, n) over the CTA, MAP_BATCH independent loads per thread issued before their stores (a
// plain loop would wait out each global or DSMEM load's latency in turn)
template <typename Load, typename Store>
__device__ __forceinline__ void map_copy(int n, Load load, Store store) {
    for (int i0 = threadIdx.x; i0 < n; i0 += ENC_TPB * MAP_BATCH) {
        float v[MAP_BATCH];
#pragma unroll
        for (int u = 0; u < MAP_BATCH; ++u) {
            const int i = i0 + u * ENC_TPB;
            v[u] = i < n ? load(i) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < MAP_BATCH; ++u) {
            const int i = i0 + u * ENC_TPB;
            if (i < n) store(i, v[u]);
        }
    }
}

// floats before the conv2 slice s2: max(conv1 rows + max(conv1 phase, conv2 phase), conv3 phase).  T = double on the
// host for the limit check (no overflow at any argument), int in the kernel (the check has passed).
template <typename T>
__host__ __device__ __forceinline__ T map_region(const MapParams& p) {
    const EncLayer &L1 = p.l[0], &L2 = p.l[1], &L3 = p.l[2];
    const T rows1 = (T)L1.oc * ((L1.ho + ENC_CL - 1) / ENC_CL) * L1.wo;
    const T ph1 = (T)L1.oc * p.C * L1.kh * L1.kw + (T)p.C * L1.kh * p.W;
    const T ph2 = (T)L1.oc * L2.kh * L1.wo + (T)enc_chunk(L2.oc) * L1.oc * L2.kh * L2.kw;
    const T ph3 = (T)L2.oc * L2.ho * L2.wo + (T)enc_chunk(L3.oc) * L2.oc * L3.kh * L3.kw;
    const T a = rows1 + (ph1 > ph2 ? ph1 : ph2);
    return a > ph3 ? a : ph3;
}

// floats of a rank's conv2 slice
template <typename T>
__host__ __device__ __forceinline__ T map_slice2(const MapParams& p) {
    return (T)enc_chunk(p.l[1].oc) * p.l[1].ho * p.l[1].wo;
}

// grid (ENC_CL, B), cluster (ENC_CL, 1, 1), block ENC_TPB; dynamic smem (map_region + map_slice2) floats.  KW1_ > 0
// fixes conv1's kernel width and K2_ > 0 conv2's kernel size at compile time (the reference's gm 8 / 4 x 4 and am 5 /
// 3 x 3: the tap loops unroll); 0 reads them from p.  The arithmetic is the same either way.
template <int KW1_, int K2_>
__global__ void __cluster_dims__(ENC_CL, 1, 1) __launch_bounds__(ENC_TPB)
map_encoder_conv_kernel(const MapParams p, float* __restrict__ feat) {
    extern __shared__ float enc_smem[];
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = (int)cluster.block_rank(), n = blockIdx.y, tid = threadIdx.x;
    const EncLayer &L1 = p.l[0], &L2 = p.l[1], &L3 = p.l[2];
    const int IC = p.C, KH = L1.kh, KW = KW1_ > 0 ? KW1_ : L1.kw, K1 = IC * KH * KW, C1 = L1.oc, W1 = L1.wo;
    const int NR1 = (L1.ho + ENC_CL - 1) / ENC_CL;          // conv1 rows per rank
    const int KH2 = K2_ > 0 ? K2_ : L2.kh, KW2 = K2_ > 0 ? K2_ : L2.kw, W2 = L2.wo, HW2 = L2.ho * W2;
    float* a1 = enc_smem;                                    // [C1][NR1][W1]: conv1 rows rank, rank + ENC_CL, ...
    float* w1 = a1 + C1 * NR1 * W1;                          // conv1 only: [K1][C1]
    float* xs = w1 + C1 * K1;                                // conv1 only: [IC][KH][W], one output row's input rows
    float* g2 = w1;                                          // conv2 only: [C1][KH2][W1], one output row's input rows
    float* ws2 = g2 + C1 * KH2 * W1;                         // conv2 only: this rank's conv2 weight slice
    float* a2 = enc_smem;                                    // conv3 only: [C2][H2][W2]
    float* ws3 = a2 + L2.oc * HW2;                           // conv3 only: this rank's conv3 weight slice
    float* s2 = enc_smem + map_region<int>(p);               // this rank's conv2 channels [c0, c1): [c1 - c0][H2][W2]
    for (int i = tid; i < C1 * K1; i += ENC_TPB) w1[(i % K1) * C1 + i / K1] = __ldg(L1.w + i);
    const float* __restrict__ src = p.map + (long long)n * p.H * p.W * IC;
    const int npg = (W1 + MAP_PIX - 1) / MAP_PIX, row_elems = KH * p.W * IC;
    for (int oh = rank; oh < L1.ho; oh += ENC_CL) {
        __syncthreads();                                     // w1 staged; the previous row's xs is consumed
        const float* __restrict__ rows = src + (long long)oh * L1.sh * p.W * IC;
        map_copy(row_elems, [&](int i) { return __ldg(rows + i); }, [&](int i, float v) {
            const int c = i % IC, col = (i / IC) % p.W, kh = i / (IC * p.W);
            xs[(c * KH + kh) * p.W + col] = v;
        });
        __syncthreads();
        float* __restrict__ dst1 = a1 + (oh / ENC_CL) * W1;
        for (int idx = tid; idx < C1 * npg; idx += ENC_TPB) {
            const int oc = idx % C1, ow0 = (idx / C1) * MAP_PIX, nvalid = min(MAP_PIX, W1 - ow0);
            int xo[MAP_PIX];
            float acc[MAP_PIX];
            const float b = L1.b ? __ldg(L1.b + oc) : 0.f;
#pragma unroll
            for (int t = 0; t < MAP_PIX; ++t) {
                xo[t] = (ow0 + min(t, nvalid - 1)) * L1.sw;  // the tail of a row recomputes its last pixel
                acc[t] = b;
            }
            for (int c = 0; c < IC; ++c)
                for (int kh = 0; kh < KH; ++kh) {
                    const float* __restrict__ xr = xs + (c * KH + kh) * p.W;
                    const float* __restrict__ wr = w1 + ((c * KH + kh) * KW) * C1 + oc;
#pragma unroll
                    for (int kw = 0; kw < KW; ++kw) {
                        const float w = wr[kw * C1];
#pragma unroll
                        for (int t = 0; t < MAP_PIX; ++t) acc[t] = fmaf(xr[xo[t] + kw], w, acc[t]);
                    }
                }
#pragma unroll
            for (int t = 0; t < MAP_PIX; ++t) {
                if (t >= nvalid) break;
                dst1[oc * NR1 * W1 + ow0 + t] = L1.relu ? relu_keep_nan(acc[t]) : acc[t];
            }
        }
    }
    int c0, c1;
    enc_slice(L2.oc, rank, c0, c1);
    __syncthreads();                                         // this CTA is done with w1 / xs
    enc_stage_weights(ws2, L2.w, c0, c1, C1 * KH2 * KW2);
    cluster.sync();                                          // every rank's conv1 rows are complete
    for (int oh2 = 0; oh2 < L2.ho; ++oh2) {
        map_copy(C1 * KH2 * W1, [&](int i) {
            const int col = i % W1, kh = (i / W1) % KH2, ic = i / (KH2 * W1), ih = oh2 * L2.sh + kh;
            return *cluster.map_shared_rank(a1 + (ic * NR1 + ih / ENC_CL) * W1 + col, ih % ENC_CL);
        }, [&](int i, float v) { g2[i] = v; });
        __syncthreads();
        for (int idx = tid; idx < (c1 - c0) * W2; idx += ENC_TPB) {
            const int oc = c0 + idx / W2, ow = idx % W2;
            const float* __restrict__ w = ws2 + (oc - c0) * C1 * KH2 * KW2;
            const float* __restrict__ x0 = g2 + ow * L2.sw;
            float acc = L2.b ? __ldg(L2.b + oc) : 0.f;
            for (int ic = 0; ic < C1; ++ic)
#pragma unroll
                for (int kh = 0; kh < KH2; ++kh) {
                    const float* __restrict__ x = x0 + (ic * KH2 + kh) * W1;
                    const float* __restrict__ wr = w + (ic * KH2 + kh) * KW2;
#pragma unroll
                    for (int kw = 0; kw < KW2; ++kw) acc = fmaf(x[kw], wr[kw], acc);
                }
            s2[(oc - c0) * HW2 + oh2 * W2 + ow] = L2.relu ? relu_keep_nan(acc) : acc;
        }
        __syncthreads();                                     // g2 is consumed
    }
    cluster.sync();                                          // every conv2 slice is complete; nobody reads a1 any more
    const int chunk2 = enc_chunk(L2.oc);
    map_copy(L2.oc * HW2, [&](int i) {
        const int owner = i / HW2 / chunk2;
        return *cluster.map_shared_rank(s2 + (i - owner * chunk2 * HW2), owner);
    }, [&](int i, float v) { a2[i] = v; });
    enc_slice(L3.oc, rank, c0, c1);
    enc_stage_weights(ws3, L3.w, c0, c1, L2.oc * L3.kh * L3.kw);
    cluster.sync();                                          // a2 is complete; no DSMEM access after this
    const long long F = (long long)L3.oc * L3.ho * L3.wo;
    enc_conv_layer(cluster, rank, a2, L2.oc, L2.ho, L2.wo, L3, ws3, nullptr, feat + n * F);
}

// ---------------------------------------------------------------------------
// One nn.GRU step (one layer, with bias) on masked state, RNNStateEncoder.single_forward
// (ss_baselines/av_nav/models/rnn_state_encoder.py:80-90): h = m h_prev, then torch's gate equations in r, z, n row
// order.  Bound by weight traffic at rollout batch sizes, so it is tiled as audio_encoder_linear_kernel: a CTA owns
// hidden unit j (its three rows of W_ih and of W_hh) for a tile of LIN_ENVS envs and streams each of those rows once;
// lane l of warp w sums the columns f = l + 32 (w + LIN_WARPS k) in increasing k, the lanes are combined by a butterfly
// and the warps in warp order.  The gate arithmetic runs in the epilogue with full-precision expf / tanhf.
// ---------------------------------------------------------------------------
// red[w][g LIN_ENVS + e] = warp w's share of sum_f W[g Hd + j][f] v[e0 + e][f], v = x, or m h when m != nullptr
__device__ __forceinline__ void gru_gate_sums(const float* __restrict__ v, const float* __restrict__ m, int ne, int K,
                                              const float* __restrict__ w, long long gate_stride,
                                              float (*red)[3 * LIN_ENVS]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float acc[3][LIN_ENVS];
#pragma unroll
    for (int g = 0; g < 3; ++g)
#pragma unroll
        for (int e = 0; e < LIN_ENVS; ++e) acc[g][e] = 0.f;
    for (int f = warp * 32 + lane; f < K; f += 32 * LIN_WARPS) {
        float wg[3];
#pragma unroll
        for (int g = 0; g < 3; ++g) wg[g] = __ldg(w + g * gate_stride + f);
#pragma unroll
        for (int e = 0; e < LIN_ENVS; ++e) {
            const int ee = min(e, ne - 1);                   // envs past B: not stored
            float xv = __ldg(v + (long long)ee * K + f);
            if (m) xv = __ldg(m + ee) * xv;
#pragma unroll
            for (int g = 0; g < 3; ++g) acc[g][e] = fmaf(wg[g], xv, acc[g][e]);
        }
    }
#pragma unroll
    for (int g = 0; g < 3; ++g)
#pragma unroll
        for (int e = 0; e < LIN_ENVS; ++e)
#pragma unroll
            for (int s = 16; s >= 1; s >>= 1) acc[g][e] += __shfl_xor_sync(0xffffffffu, acc[g][e], s);
#pragma unroll
    for (int g = 0; g < 3; ++g)
#pragma unroll
        for (int e = 0; e < LIN_ENVS; ++e)
            if (lane == ((g * LIN_ENVS + e) & 31)) red[warp][g * LIN_ENVS + e] = acc[g][e];
}

__device__ __forceinline__ float gru_sigmoid(float a) { return 1.f / (1.f + expf(-a)); }

// grid (Hd, ceil(B / LIN_ENVS)), block 32 LIN_WARPS
__global__ void __launch_bounds__(32 * LIN_WARPS)
gru_step_kernel(const float* __restrict__ x, const float* __restrict__ h, const float* __restrict__ masks, int B, int I,
                int Hd, const float* __restrict__ w_ih, const float* __restrict__ w_hh, const float* __restrict__ b_ih,
                const float* __restrict__ b_hh, float* __restrict__ out, float* __restrict__ h_out) {
    __shared__ float red_i[LIN_WARPS][3 * LIN_ENVS], red_h[LIN_WARPS][3 * LIN_ENVS];
    const int j = blockIdx.x, e0 = blockIdx.y * LIN_ENVS, ne = min(LIN_ENVS, B - e0);
    gru_gate_sums(x + (long long)e0 * I, nullptr, ne, I, w_ih + (long long)j * I, (long long)Hd * I, red_i);
    gru_gate_sums(h + (long long)e0 * Hd, masks + e0, ne, Hd, w_hh + (long long)j * Hd, (long long)Hd * Hd, red_h);
    __syncthreads();
    const int e = threadIdx.x;
    if (e >= ne) return;
    float gi[3], gh[3];
#pragma unroll
    for (int g = 0; g < 3; ++g) {
        float si = red_i[0][g * LIN_ENVS + e], sh = red_h[0][g * LIN_ENVS + e];
#pragma unroll
        for (int w = 1; w < LIN_WARPS; ++w) {
            si += red_i[w][g * LIN_ENVS + e];
            sh += red_h[w][g * LIN_ENVS + e];
        }
        gi[g] = si + __ldg(b_ih + g * Hd + j);
        gh[g] = sh + __ldg(b_hh + g * Hd + j);
    }
    const long long o = (long long)(e0 + e) * Hd + j;
    const float r = gru_sigmoid(gi[0] + gh[0]);
    const float z = gru_sigmoid(gi[1] + gh[1]);
    const float nn = tanhf(gi[2] + r * gh[2]);
    const float hp = __ldg(masks + e0 + e) * __ldg(h + o);
    const float hn = (1.f - z) * nn + z * hp;
    out[o] = hn;
    h_out[o] = hn;
}

// ---------------------------------------------------------------------------
// RNNStateEncoder.seq_forward (ss_baselines/av_nav/models/rnn_state_encoder.py:92-143) and its backward, for PPO's
// update.  The carried state is multiplied by masks[t] only at a segment start: t = 0, or a t >= 1 at which some env's
// mask is 0.0 (the reference's split points, decided here on the device from the masks).  Three kernels:
//   gru_gemm_kernel<TA, TB>   C = op(A) op(B) (+ bias per column), optional sums of op(A)'s rows: the input projection
//                             X W_ih^T + b_ih, dX = dG_i W_ih, dW_ih = dG_i^T X (+ db_ih), dW_hh = dG_h^T H_prev (+ db_hh)
//   gru_seq_fwd_kernel        the forward recurrence, one grid.sync per step
//   gru_seq_bwd_kernel        the reverse recurrence, one grid.sync per step
// The recurrences are cooperative launches of at most one CTA per SM.  CTA c owns hidden units [c U, c U + U) for the
// whole sequence and keeps their W_hh slice in shared memory: forward its 3 U rows (h-gate sums), backward the same
// rows read as columns (W_hh^T dG_h).  A step's new state (forward) or gate gradients (backward) of every unit are in
// global memory after the step's grid.sync; everything else a CTA needs at the next step it wrote itself.  Every sum
// runs in an order fixed by the shapes: each (env, unit) gate sum is one warp's, lane l over k = l + 32 i in increasing
// i, then a butterfly; GEMM k loops run in increasing k.  No float atomics, so results are deterministic, and an env's
// out, h_last, dx and dh0 do not depend on N or on its position.
// ---------------------------------------------------------------------------
constexpr int GG_BM = 64, GG_BN = 64, GG_BK = 16, GG_THREADS = 256;   // GEMM tile, 4 x 4 outputs per thread
constexpr int GS_THREADS = 256, GS_WARPS = GS_THREADS / 32;             // recurrence CTA
constexpr int GS_SMEM_MAX = 232448;                                     // sm_90 opt-in shared memory per CTA

// C[m][n] = sum_k A(m, k) B(k, n) (+ bias[n]) for m < M, n < Nc; A(m, k) = A[m lda + k], or A[k lda + m] when TA;
// B(k, n) = B[k ldb + n], or B[n ldb + k] when TB.  C may be NULL; rowsum[m] = sum_k A(m, k) is written by the CTAs of
// column tile 0 when rowsum is not NULL.  grid (ceil(Nc / 64), ceil(M / 64)).
template <bool TA, bool TB>
__global__ void __launch_bounds__(GG_THREADS)
gru_gemm_kernel(int M, int Nc, int K, const float* __restrict__ A, long long lda, const float* __restrict__ B,
                long long ldb, const float* __restrict__ bias, float* __restrict__ C, long long ldc,
                float* __restrict__ rowsum) {
    __shared__ float As[GG_BK][GG_BM], Bs[GG_BK][GG_BN];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int m0 = blockIdx.y * GG_BM, n0 = blockIdx.x * GG_BN;
    const bool sums = rowsum && blockIdx.x == 0;
    float acc[4][4] = {}, rs[4] = {};
    for (int k0 = 0; k0 < K; k0 += GG_BK) {
#pragma unroll
        for (int i = 0; i < GG_BM * GG_BK / GG_THREADS; ++i) {
            const int idx = tid + GG_THREADS * i;
            const int m = TA ? idx % GG_BM : idx / GG_BK, k = TA ? idx / GG_BM : idx % GG_BK;
            const int gm = m0 + m, gk = k0 + k;
            As[k][m] = gm < M && gk < K ? __ldg(A + (TA ? (long long)gk * lda + gm : (long long)gm * lda + gk)) : 0.f;
            const int n = TB ? idx / GG_BK : idx % GG_BN, kb = TB ? idx % GG_BK : idx / GG_BN;
            const int gn = n0 + n, gkb = k0 + kb;
            Bs[kb][n] = gn < Nc && gkb < K ? __ldg(B + (TB ? (long long)gn * ldb + gkb : (long long)gkb * ldb + gn)) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < GG_BK; ++k) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[k][ty + 16 * i];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = Bs[k][tx + 16 * j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
            if (sums) {
#pragma unroll
                for (int i = 0; i < 4; ++i) rs[i] += a[i];
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty + 16 * i;
        if (m >= M) continue;
        if (sums && tx == 0) rowsum[m] = rs[i];
        if (!C) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx + 16 * j;
            if (n < Nc) C[(long long)m * ldc + n] = bias ? acc[i][j] + __ldg(bias + n) : acc[i][j];
        }
    }
}

// t = 0, or some env's masks[t] is 0.0 (NaN is not): the reference's has_zeros.  Every thread of the CTA gets it.
__device__ __forceinline__ bool gru_segment_start(const float* __restrict__ masks, int t, int N) {
    bool z = t == 0;
    if (!z)
        for (int e = threadIdx.x; e < N; e += blockDim.x) z = z || __ldg(masks + (long long)t * N + e) == 0.f;
    return __syncthreads_or(z) != 0;
}

struct GruSeqArgs {
    const float* masks;     // [T][N]
    const float* w_hh;      // [3 Hd][Hd]
    const float* b_hh;      // [3 Hd]
    const float* h0;        // [N][Hd]
    const float* gi;        // [T N][3 Hd]: X W_ih^T + b_ih (forward)
    float* out;             // [T N][Hd]
    float* h_last;          // [N][Hd]
    float* saved;           // [5][T N][Hd]: H_prev, r, z, n, W_hn H_prev + b_hn; NULL: not saved
    const float* dout;      // [T N][Hd] or NULL (backward)
    const float* dh_last;   // [N][Hd] or NULL
    float* dgi;             // [T N][3 Hd] gradient of X W_ih^T + b_ih
    float* dgh;             // [T N][3 Hd] gradient of W_hh H_prev + b_hh
    float* dh0;             // [N][Hd] or NULL
    int T, N, Hd, U;        // U hidden units per CTA
    int E;                  // envs per shared-memory chunk of the step's operand rows
};

// Each step's operand rows (forward: the N previous states, backward: the N rows of dG_h) are read from L2 by a
// whole CTA at once, E envs at a time, into shared memory; the per-(env, unit) sums then run from shared memory.
constexpr int GS_STAGE_FLOATS = 16384;

// dynamic smem: ws[3 U][Hd] (row g U + u = W_hh row g Hd + j0 + u), hsm[E][Hd] (masked previous states of E envs),
// gis[E][3][U] (their input projections of the owned units)
__global__ void __launch_bounds__(GS_THREADS) gru_seq_fwd_kernel(const GruSeqArgs a) {
    extern __shared__ float ws[];
    cg::grid_group grid = cg::this_grid();
    const int T = a.T, N = a.N, Hd = a.Hd, U = a.U, E = a.E;
    const int j0 = blockIdx.x * U, nu = min(U, Hd - j0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* hsm = ws + (long long)3 * U * Hd;
    float* gis = hsm + (long long)E * Hd;
    for (int i = threadIdx.x; i < 3 * U * Hd; i += GS_THREADS) {
        const int row = i / Hd, g = row / U, u = row % U, k = i % Hd;
        ws[i] = u < nu ? __ldg(a.w_hh + (long long)(g * Hd + j0 + u) * Hd + k) : 0.f;
    }
    const long long TN = (long long)T * N, plane = TN * Hd;
    for (int t = 0; t < T; ++t) {
        const bool seg = gru_segment_start(a.masks, t, N);   // also a CTA barrier
        const float* hs = t == 0 ? a.h0 : a.out + (long long)(t - 1) * N * Hd;   // written by the previous step
        for (int e0 = 0; e0 < N; e0 += E) {
            const int ne = min(E, N - e0);
            const float* src = hs + (long long)e0 * Hd;
            for (int i = threadIdx.x; i < ne * Hd; i += GS_THREADS) {
                const float v = __ldcg(src + i);
                hsm[i] = seg ? __ldg(a.masks + (long long)t * N + e0 + i / Hd) * v : v;
            }
            for (int i = threadIdx.x; i < ne * 3 * nu; i += GS_THREADS) {
                const int e = i / (3 * nu), g = i % (3 * nu) / nu, u = i % nu;
                gis[(e * 3 + g) * U + u] = __ldg(a.gi + ((long long)t * N + e0 + e) * 3 * Hd + g * Hd + j0 + u);
            }
            __syncthreads();
            for (int p = warp; p < ne * nu; p += GS_WARPS) {
                const int el = p / nu, u = p % nu, e = e0 + el, j = j0 + u;
                const float* he = hsm + (long long)el * Hd;
                const float* w0 = ws + (long long)u * Hd;
                float s[3] = {0.f, 0.f, 0.f};
                for (int k = lane; k < Hd; k += 32) {
                    const float hv = he[k];
#pragma unroll
                    for (int g = 0; g < 3; ++g) s[g] = fmaf(w0[(long long)g * U * Hd + k], hv, s[g]);
                }
#pragma unroll
                for (int g = 0; g < 3; ++g)
#pragma unroll
                    for (int o = 16; o >= 1; o >>= 1) s[g] += __shfl_xor_sync(0xffffffffu, s[g], o);
                if (lane == 0) {
                    const float* gi = gis + el * 3 * U + u;
                    float gh[3];
#pragma unroll
                    for (int g = 0; g < 3; ++g) gh[g] = s[g] + __ldg(a.b_hh + g * Hd + j);
                    const float r = gru_sigmoid(gi[0] + gh[0]);
                    const float z = gru_sigmoid(gi[U] + gh[1]);
                    const float nn = tanhf(gi[2 * U] + r * gh[2]);
                    const float hp = he[j];
                    const float hn = (1.f - z) * nn + z * hp;
                    const long long o = ((long long)t * N + e) * Hd + j;
                    a.out[o] = hn;
                    if (t == T - 1) a.h_last[(long long)e * Hd + j] = hn;
                    if (a.saved) {
                        a.saved[o] = hp;
                        a.saved[plane + o] = r;
                        a.saved[2 * plane + o] = z;
                        a.saved[3 * plane + o] = nn;
                        a.saved[4 * plane + o] = gh[2];
                    }
                }
            }
            __syncthreads();
        }
        if (t + 1 < T) grid.sync();
    }
}

// dynamic smem: ws[U][3 Hd] (ws[u][k] = W_hh[k][j0 + u]), c[N][U] (the carried gradient of each owned unit),
// gsm[E][3 Hd] (rows of dG_h)
__global__ void __launch_bounds__(GS_THREADS) gru_seq_bwd_kernel(const GruSeqArgs a) {
    extern __shared__ float ws[];
    cg::grid_group grid = cg::this_grid();
    const int T = a.T, N = a.N, Hd = a.Hd, U = a.U, E = a.E, K3 = 3 * Hd;
    const int j0 = blockIdx.x * U, nu = min(U, Hd - j0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* c = ws + (long long)U * K3;
    float* gsm = c + (long long)N * U;
    for (int i = threadIdx.x; i < U * K3; i += GS_THREADS) {
        const int u = i / K3, k = i % K3;
        ws[i] = u < nu ? __ldg(a.w_hh + (long long)k * Hd + j0 + u) : 0.f;
    }
    for (int i = threadIdx.x; i < N * U; i += GS_THREADS) c[i] = 0.f;
    __syncthreads();
    const long long TN = (long long)T * N, plane = TN * Hd;
    for (int t = T - 1; t >= 0; --t) {
        // gate gradients of the owned units; c becomes z dh, the direct part of dh_prev
        for (int p = threadIdx.x; p < N * nu; p += GS_THREADS) {
            const int e = p / nu, u = p % nu, j = j0 + u;
            const long long row = (long long)t * N + e, o = row * Hd + j;
            float dh = c[e * U + u];
            if (a.dout) dh += __ldg(a.dout + o);
            if (t == T - 1 && a.dh_last) dh += __ldg(a.dh_last + (long long)e * Hd + j);
            const float hp = __ldg(a.saved + o), r = __ldg(a.saved + plane + o), z = __ldg(a.saved + 2 * plane + o);
            const float nn = __ldg(a.saved + 3 * plane + o), ghn = __ldg(a.saved + 4 * plane + o);
            const float dn = dh * (1.f - z), dz = dh * (hp - nn);
            const float dan = dn * (1.f - nn * nn);
            const float dar = dan * ghn * r * (1.f - r);
            const float daz = dz * z * (1.f - z);
            float* gi = a.dgi + row * K3;
            float* gh = a.dgh + row * K3;
            gi[j] = dar;
            gi[Hd + j] = daz;
            gi[2 * Hd + j] = dan;
            gh[j] = dar;
            gh[Hd + j] = daz;
            gh[2 * Hd + j] = dan * r;
            c[e * U + u] = dh * z;
        }
        const bool seg = gru_segment_start(a.masks, t, N);   // also orders c's writes before the reads below
        grid.sync();
        // dh_prev = z dh + W_hh^T dG_h, times masks[t] at a segment start
        for (int e0 = 0; e0 < N; e0 += E) {
            const int ne = min(E, N - e0);
            const float* src = a.dgh + ((long long)t * N + e0) * K3;   // written by every CTA before the grid.sync
#pragma unroll 4
            for (int i = threadIdx.x; i < ne * K3; i += GS_THREADS) gsm[i] = __ldcg(src + i);
            __syncthreads();
            for (int p = warp; p < ne * nu; p += GS_WARPS) {
                const int el = p / nu, u = p % nu, e = e0 + el;
                const float* g = gsm + (long long)el * K3;
                const float* w = ws + (long long)u * K3;
                float s = 0.f;
                for (int k = lane; k < K3; k += 32) s = fmaf(w[k], g[k], s);
#pragma unroll
                for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                if (lane == 0) {
                    const float dhp = c[e * U + u] + s;
                    const float v = seg ? __ldg(a.masks + (long long)t * N + e) * dhp : dhp;
                    c[e * U + u] = v;
                    if (t == 0 && a.dh0) a.dh0[(long long)e * Hd + j0 + u] = v;
                }
            }
            __syncthreads();
        }
    }
}

// ---------------------------------------------------------------------------
// The CNN encoders' conv stack for PPO's update: AudioCNN, VisualCNN and MapCNN (Conv2d ReLU Conv2d ReLU Conv2d Flatten
// Linear ReLU, unpadded) forward and backward on minibatches of thousands of envs.  Each conv is one implicit GEMM,
// cs_gemm_kernel, tiled across envs instead of one env per cluster:
//   CS_FWD  out[(n, pos)][oc] = bias + sum_k X[(n, pos)][k] W[oc][k]: a 128 (env, output pixel) x 32 channel tile, 4 x 4
//           outputs per thread, each a single fmaf chain over k in the order of the inference kernels (bias, then
//           (ic, kh, kw); the spectrogram's conv1 (kh, kw, ear) as conv1_point; SAVi's folded label bias as the
//           start), so features and out are bit-identical to ssb_{audio,visual,map}_encoder_batch.
//   CS_DW   dW[oc][k] = sum over (n, pos) of G[(n, pos)][oc] X[(n, pos)][k], and db: one partial sum per chunk of
//           CS_RCHUNK rows, summed over the chunks in order by cs_reduce_kernel.  No float atomics.
//   CS_DX   dX of the layer input as a gather-form transposed conv.  Input pixels are grouped by their residue
//           (ih mod SH, iw mod SW), so a tile only enumerates the taps that can reach it: k = (oc, jh, jw) with
//           kh = ih mod SH + SH jh.  An env's dX is a fixed sum of its own G, whatever B and its position.
// X is the im2col view of the layer input, read through a per-column table in shared memory; G is the gradient of the
// layer output, masked as torch's threshold_backward does (0 where the ReLU output is <= 0; NaN passes).
// ---------------------------------------------------------------------------
constexpr int CS_BM = 128, CS_BN = 32, CS_BK = 16, CS_THREADS = 256;
constexpr int CS_RCHUNK = 2048;                  // weight gradients: rows (env, output pixel) per partial sum
enum { CS_FWD = 0, CS_DW = 1, CS_DX = 2 };

struct CsLayer {
    // layer input: kind 0 a channels-first [B][IC][H][W] activation in x; kind 1 conv1 from channels-last x [B][H][W][nA]
    // (times 1 / 255 when scale) and x2 [B][H][W][nB] with k = (ic, kh, kw); kind 2 the same with k = (kh, kw, ic), the
    // spectrogram's ear order (conv1_point)
    int kind, B, IC, H, W, nA, nB, scale;
    const float* x;
    const float* x2;
    int OC, KH, KW, SH, SW, Ho, Wo, relu;
    int Kw, K;                                   // floats per weight row; GEMM columns (CS_DX: the most of any class)
    const float* w;
    const float* bias;
    const float* lbias;                          // [B][OC] conv1 bias with SAVi's labels folded in, or NULL
    const float* g;                              // gradient of the layer output [B][OC][Ho][Wo]
    const float* gmask;                          // the layer output, for the ReLU mask when grelu
    int grelu;
    int xrelu;                                   // CS_DX: mask dX where the input activation x is <= 0
    float* out;                                  // CS_FWD [B][OC][Ho][Wo]; CS_DX [B][IC][H][W]
    float* part;                                 // CS_DW [chunks][OC][K] and [chunks][OC]
    float* partb;
};

// input offset, channel and weight-row index of GEMM column k (CS_FWD, CS_DW)
__device__ __forceinline__ void cs_col(const CsLayer& L, int k, int& off, int& ch, int& wi) {
    const int KK = L.KH * L.KW;
    const int ic = L.kind == 2 ? k % L.IC : k / KK, t = L.kind == 2 ? k / L.IC : k % KK;
    const int kh = t / L.KW, kw = t % L.KW;
    wi = ic * KK + t;
    off = L.kind == 0 ? (ic * L.H + kh) * L.W + kw : kh * L.W + kw;
    ch = ic;
}

template <bool CL>
__device__ __forceinline__ float cs_x(const CsLayer& L, int base, int off, int ch) {
    if (!CL) return __ldg(L.x + base + off);
    const long long p = (long long)base + off;
    if (ch < L.nA) {
        const float v = __ldg(L.x + p * L.nA + ch);
        return L.scale ? v * (1.0f / 255.0f) : v;                  // torch's CUDA x / 255.0, as the inference kernel
    }
    return __ldg(L.x2 + p * L.nB + (ch - L.nA));
}

__device__ __forceinline__ float cs_g(const CsLayer& L, int i) {
    const float g = __ldg(L.g + i);
    return L.grelu && __ldg(L.gmask + i) <= 0.f ? 0.f : g;
}

// grid CS_FWD (ceil(B Ho Wo / 128), ceil(OC / 32)); CS_DW (chunks, ceil(K / 128), ceil(OC / 32)); CS_DX
// (ceil(B ceil(H / SH) ceil(W / SW) / 128), ceil(IC / 32), SH SW).  Dynamic smem 4 K ints.  CL: the layer input is
// conv1's channels-last observation (kind 1 or 2), else a channels-first activation (kind 0).  A warp covers 8 x 4
// threads of 4 x 4 outputs, so a step's shared-memory reads are 2 + 1 wavefronts per 16 FMA per thread.  The global
// loads of the next K tile are issued before the current tile's FMAs.
template <int MODE, bool CL>
__global__ void __launch_bounds__(CS_THREADS, 3) cs_gemm_kernel(const __grid_constant__ CsLayer L) {
    extern __shared__ int cs_tab[];
    __shared__ __align__(16) float As[CS_BK][CS_BM + 4];
    __shared__ __align__(16) float Bs[CS_BK][CS_BN + 4];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tr = (warp & 3) * 8 + (lane & 7), tc = (warp >> 2) * 4 + (lane >> 3);
    const int HWo = L.Ho * L.Wo, KK = L.KH * L.KW;
    int* t0 = cs_tab;
    int* t1 = cs_tab + L.K;
    int* t2 = cs_tab + 2 * L.K;
    int* t3 = cs_tab + 3 * L.K;
    // the tile: M output rows from m0, columns from c0 (Nc of them), reduction over [r0, r1)
    int M, r0 = 0, r1, m0, c0, Nc;
    int rh = 0, rw = 0, Qh = 0, Qw = 0;
    if (MODE == CS_FWD) {
        M = L.B * HWo; r1 = L.K; m0 = blockIdx.x * CS_BM; c0 = blockIdx.y * CS_BN; Nc = L.OC;
        for (int k = tid; k < L.K; k += CS_THREADS) cs_col(L, k, t0[k], t1[k], t2[k]);
    } else if (MODE == CS_DW) {
        M = L.K; r0 = blockIdx.x * CS_RCHUNK; r1 = min(L.B * HWo, r0 + CS_RCHUNK); m0 = blockIdx.y * CS_BM;
        c0 = blockIdx.z * CS_BN; Nc = L.OC;
        for (int k = tid; k < L.K; k += CS_THREADS) cs_col(L, k, t0[k], t1[k], t2[k]);
    } else {
        rh = blockIdx.z / L.SW; rw = blockIdx.z % L.SW;
        Qh = (L.H - rh + L.SH - 1) / L.SH; Qw = (L.W - rw + L.SW - 1) / L.SW;
        const int Jh = rh < L.KH ? (L.KH - rh + L.SH - 1) / L.SH : 0, Jw = rw < L.KW ? (L.KW - rw + L.SW - 1) / L.SW : 0;
        M = L.B * Qh * Qw; r1 = L.OC * Jh * Jw; m0 = blockIdx.x * CS_BM; c0 = blockIdx.y * CS_BN; Nc = L.IC;
        for (int k = tid; k < r1; k += CS_THREADS) {
            const int oc = k / (Jh * Jw), jh = (k / Jw) % Jh, jw = k % Jw;
            t0[k] = oc * HWo - jh * L.Wo - jw;
            t1[k] = jh;
            t2[k] = jw;
            t3[k] = oc * L.Kw + (rh + L.SH * jh) * L.KW + rw + L.SW * jw;
        }
        if (m0 >= M) return;                             // a smaller residue class
    }
    __syncthreads();
    // CS_FWD / CS_DX: this thread loads output row am of the tile at steps ak + 2 i.  CS_DW: reduction row ar of the
    // tile, at GEMM columns ak + 16 i and gradient columns ak + 16 i.
    const int am = tid % CS_BM, ak2 = tid / CS_BM, ar = tid % CS_BK, ak = tid / CS_BK;
    int abase = 0, aq0 = 0, aq1 = 0;
    bool arow = false;
    if (MODE == CS_FWD) {
        arow = m0 + am < M;
        if (arow) {
            const int m = m0 + am, n = m / HWo, pos = m - n * HWo, oh = pos / L.Wo, ow = pos - oh * L.Wo;
            abase = ((CL ? n * L.H : n * L.IC * L.H) + oh * L.SH) * L.W + ow * L.SW;
        }
    } else if (MODE == CS_DX) {
        arow = m0 + am < M;
        if (arow) {
            const int m = m0 + am, n = m / (Qh * Qw), q = m - n * Qh * Qw;
            aq0 = q / Qw;
            aq1 = q - aq0 * Qw;
            abase = n * L.OC * HWo + aq0 * L.Wo + aq1;
        }
    }
    float ra[8], rb[2];
    auto load = [&](int k0) {
        const int nk = min(CS_BK, r1 - k0);
        if (MODE == CS_DW) {
            const int r = k0 + ar;
            int xb = 0, gb = 0;
            if (ar < nk) {
                const int n = r / HWo, pos = r - n * HWo, oh = pos / L.Wo, ow = pos - oh * L.Wo;
                xb = ((CL ? n * L.H : n * L.IC * L.H) + oh * L.SH) * L.W + ow * L.SW;
                gb = n * L.OC * HWo + pos;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int k = m0 + ak + 16 * i;
                ra[i] = ar < nk && k < L.K ? cs_x<CL>(L, xb, t0[k], t1[k]) : 0.f;
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int oc = c0 + ak + 16 * i;
                rb[i] = ar < nk && oc < Nc ? cs_g(L, gb + oc * HWo) : 0.f;
            }
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int kk = ak2 + 2 * i, k = k0 + kk;
                float v = 0.f;
                if (arow && kk < nk) {
                    if (MODE == CS_FWD) {
                        v = cs_x<CL>(L, abase, t0[k], t1[k]);
                    } else {
                        const int oh = aq0 - t1[k], ow = aq1 - t2[k];
                        if (oh >= 0 && oh < L.Ho && ow >= 0 && ow < L.Wo) v = cs_g(L, abase + t0[k]);
                    }
                }
                ra[i] = v;
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                // consecutive lanes read consecutive k of one column: contiguous weights
                const int e = tid + CS_THREADS * i, kk = e % CS_BK, col = c0 + e / CS_BK, k = k0 + kk;
                float v = 0.f;
                if (kk < nk && col < Nc)
                    v = MODE == CS_FWD ? __ldg(L.w + (long long)col * L.Kw + t2[k]) : __ldg(L.w + t3[k] + col * KK);
                rb[i] = v;
            }
        }
    };
    auto store = [&]() {
        if (MODE == CS_DW) {
#pragma unroll
            for (int i = 0; i < 8; ++i) As[ar][ak + 16 * i] = ra[i];
#pragma unroll
            for (int i = 0; i < 2; ++i) Bs[ar][ak + 16 * i] = rb[i];
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) As[ak2 + 2 * i][am] = ra[i];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int e = tid + CS_THREADS * i;
                Bs[e % CS_BK][e / CS_BK] = rb[i];
            }
        }
    };
    float acc[4][4], rs[4] = {0.f, 0.f, 0.f, 0.f};
    if (MODE == CS_FWD) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int m = min(m0 + tr * 4 + i, M - 1), n = m / HWo;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int oc = min(c0 + tc * 4 + j, Nc - 1);
                acc[i][j] = L.lbias ? __ldg(L.lbias + n * L.OC + oc) : L.bias ? __ldg(L.bias + oc) : 0.f;
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    }
    const bool sums = MODE == CS_DW && blockIdx.y == 0 && tr == 0;
    auto step = [&](int k) {
        const float4 a = *reinterpret_cast<const float4*>(&As[k][tr * 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tc * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        if (sums) {
#pragma unroll
            for (int j = 0; j < 4; ++j) rs[j] += bv[j];
        }
    };
    if (r0 < r1) load(r0);
    for (int k0 = r0; k0 < r1; k0 += CS_BK) {
        store();
        __syncthreads();
        const int nk = min(CS_BK, r1 - k0);
        if (k0 + CS_BK < r1) load(k0 + CS_BK);
        // only the nk real steps: a padded step would add +0 and could turn a -0 sum into +0
        if (nk == CS_BK) {
#pragma unroll
            for (int k = 0; k < CS_BK; ++k) step(k);
        } else {
            for (int k = 0; k < nk; ++k) step(k);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + tr * 4 + i;
        if (MODE != CS_DW && m >= M) continue;
        // the row's output address for column 0 and the stride between columns
        long long o0 = 0, cstride = 0;
        if (MODE == CS_FWD) {
            const int n = m / HWo;
            o0 = (long long)n * L.OC * HWo + (m - n * HWo);
            cstride = HWo;
        } else if (MODE == CS_DX) {
            const int n = m / (Qh * Qw), q = m - n * Qh * Qw, qh = q / Qw;
            o0 = ((long long)n * L.IC * L.H + rh + L.SH * qh) * L.W + rw + L.SW * (q - qh * Qw);
            cstride = (long long)L.H * L.W;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int col = c0 + tc * 4 + j;
            if (col >= Nc) continue;
            if (MODE == CS_FWD) {
                L.out[o0 + col * cstride] = L.relu ? relu_keep_nan(acc[i][j]) : acc[i][j];
            } else if (MODE == CS_DX) {
                const long long o = o0 + col * cstride;
                // the gradient of the layer below's output, masked by that layer's ReLU here once
                L.out[o] = L.xrelu && __ldg(L.x + o) <= 0.f ? 0.f : acc[i][j];
            } else {
                if (m < L.K) L.part[((long long)blockIdx.x * L.OC + col) * L.K + m] = acc[i][j];
                if (sums && i == 0) L.partb[(long long)blockIdx.x * L.OC + col] = rs[j];
            }
        }
    }
}

// dW[oc][wi(k)] and db[oc] from cs_gemm_kernel<CS_DW>'s chunk partial sums, added in chunk order; either may be NULL
__global__ void __launch_bounds__(256) cs_reduce_kernel(const CsLayer L, int chunks, float* __restrict__ dw,
                                                         float* __restrict__ db) {
    const int i = blockIdx.x * 256 + threadIdx.x, OK = L.OC * L.K;
    if (i < OK && dw) {
        const int oc = i / L.K, k = i % L.K;
        float s = L.part[i];
        for (int c = 1; c < chunks; ++c) s += L.part[(long long)c * OK + i];
        int off, ch, wi;
        cs_col(L, k, off, ch, wi);
        dw[(long long)oc * L.Kw + wi] = s;
    } else if (i >= OK && i < OK + L.OC && db) {
        const int oc = i - OK;
        const float* pb = L.partb;
        float s = pb[oc];
        for (int c = 1; c < chunks; ++c) s += pb[(long long)c * L.OC + oc];
        db[oc] = s;
    }
}

// g = d_out, 0 where the Linear's ReLU output is <= 0 (NaN passes), over n floats
__global__ void __launch_bounds__(256) cs_relu_grad_kernel(const float* __restrict__ dout, const float* __restrict__ out,
                                                            int relu, int n, float* __restrict__ g) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n) g[i] = relu && __ldg(out + i) <= 0.f ? 0.f : __ldg(dout + i);
}

// lbias[n][oc] = b[oc] + sum_c labels[n][c] sum_k W1[oc][2 + c][k], in enc_fold_label_bias's order: the tap sum of a
// (channel, label) in k order, then the labels in c order by fmaf
__global__ void __launch_bounds__(256) cs_label_bias_kernel(int B, int OC, int NL, int KK, const float* __restrict__ w1,
                                                             const float* __restrict__ bias, const float* __restrict__ lab,
                                                             long long stride, float* __restrict__ lbias) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= B * OC) return;
    const int n = i / OC, oc = i % OC;
    float acc = bias ? __ldg(bias + oc) : 0.f;
    for (int c = 0; c < NL; ++c) {
        const float* t = w1 + ((long long)oc * (2 + NL) + 2 + c) * KK;
        float s = __ldg(t);
        for (int k = 1; k < KK; ++k) s += __ldg(t + k);
        acc = fmaf(__ldg(lab + n * stride + c), s, acc);
    }
    lbias[i] = acc;
}

// s[n][oc] = sum over conv1's output pixels of env n's masked gradient, in pixel order
__global__ void __launch_bounds__(256) cs_label_sum_kernel(const CsLayer L, float* __restrict__ s) {
    const int i = blockIdx.x * 256 + threadIdx.x, HWo = L.Ho * L.Wo;
    if (i >= L.B * L.OC) return;
    float acc = 0.f;
    for (int p = 0; p < HWo; ++p) acc += cs_g(L, i * HWo + p);
    s[i] = acc;
}

// A label channel is constant over every unpadded window, so each of its taps gets the same gradient:
// dW1[oc][2 + c][.] = sum_n labels[n][c] s[n][oc], in env order
__global__ void __launch_bounds__(256) cs_label_grad_kernel(int B, int OC, int NL, int KK, const float* __restrict__ lab,
                                                             long long stride, const float* __restrict__ s,
                                                             float* __restrict__ dw1) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= OC * NL) return;
    const int oc = i / NL, c = i % NL;
    float acc = 0.f;
    for (int n = 0; n < B; ++n) acc = fmaf(__ldg(lab + n * stride + c), __ldg(s + n * OC + oc), acc);
    float* t = dw1 + ((long long)oc * (2 + NL) + 2 + c) * KK;
    for (int k = 0; k < KK; ++k) t[k] = acc;
}

// ---------------------------------------------------------------------------
// The policy's action and value heads at rollout time, Policy.act after self.net (ss_baselines/av_nav/ppo/policy.py:
// 35-60, savi :42-65, av_wan :39-60): CategoricalNet / CategoricalNetWithMask (common/utils.py:58-87), CriticHead,
// CustomFixedCategorical's sample() or mode() and log_probs() (:41-55).  A CTA owns PH_ENVS envs with their features
// in shared memory; warp w computes output rows w, w + PH_WARPS, ... (row A is the critic), each weight row read
// once per tile, lane l summing columns l + 32 k in increasing k, lanes combined by a butterfly.  Then warp e runs
// env e's distribution: lane l holds actions l + 32 k, every max / sum runs over k in increasing order, then a
// butterfly.  FP32 with FMA, full-precision expf / logf.
// ---------------------------------------------------------------------------
#define PH_ENVS 4
#define PH_WARPS 16
#define PH_MAX_A 256
#define PH_MAX_H 2048
#define PH_SLOTS (PH_MAX_A / 32)

struct PolicyHeadParams {
    const float* feat;                 // [B][H]
    const float* aw;                   // [A][H]
    const float* ab;                   // [A]
    const float* cw;                   // [H]
    const float* cb;                   // [1]
    const float* mask;                 // [B][A] or NULL
    const float* q;                    // [B][A] exponential draws, NULL: mode
    float* value;                      // [B]
    long long* action;                 // [B]
    float* log_prob;                   // [B]
    float* probs;                      // [B][A] or NULL
    int* status;                       // refused rows
    int* ticket;                       // context-owned {refused so far, CTAs done}, 0 between calls
    int B, H, A, masked;
};

// torch.argmax's order: NaN above everything, then larger value, then lower index
__device__ __forceinline__ bool ph_better(float v, int i, float bv, int bi) {
    const bool vn = v != v, bn = bv != bv;
    if (vn != bn) return vn;
    if (!vn && v != bv) return v > bv;
    return i < bi;
}

__device__ __forceinline__ float ph_warp_max(float v) {
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, s));
    return v;
}

__device__ __forceinline__ float ph_warp_sum(float v) {
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

// The two stages policy_head_kernel and policy_head_train_kernel share, defined after the rollout kernel
__device__ __forceinline__ void ph_linear(const float* __restrict__ feat, const float* __restrict__ aw,
                                          const float* __restrict__ ab, const float* __restrict__ cw,
                                          const float* __restrict__ cb, int e0, int ne, int H, int A,
                                          float (*xs)[PH_MAX_H], float (*zs)[PH_MAX_A + 1]);
__device__ __forceinline__ bool ph_distribution(float* z, int masked, const float* __restrict__ mask, int n, int A,
                                                float (&v)[PH_SLOTS], float* save);

// Both head kernels' refusal count: the last CTA to finish publishes it and leaves the ticket at 0 for the next call
__device__ __forceinline__ void ph_publish(int refused, int* ticket, int* status) {
    if (threadIdx.x == 0) {
        if (refused) atomicAdd(&ticket[0], refused);
        __threadfence();
        if (atomicAdd(&ticket[1], 1) == (int)gridDim.x - 1) {
            *status = atomicExch(&ticket[0], 0);
            atomicExch(&ticket[1], 0);
        }
    }
}

// grid ceil(B / PH_ENVS), block 32 PH_WARPS
__global__ void __launch_bounds__(32 * PH_WARPS) policy_head_kernel(PolicyHeadParams p) {
    __shared__ float xs[PH_ENVS][PH_MAX_H];
    __shared__ float zs[PH_ENVS][PH_MAX_A + 1];
    __shared__ int refused;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int e0 = blockIdx.x * PH_ENVS, ne = min(PH_ENVS, p.B - e0), A = p.A;
    if (threadIdx.x == 0) refused = 0;
    ph_linear(p.feat, p.aw, p.ab, p.cw, p.cb, e0, ne, p.H, A, xs, zs);
    if (warp < ne) {
        const int n = e0 + warp;
        float v[PH_SLOTS];
        bool bad = ph_distribution(zs[warp], p.masked, p.mask, n, A, v, nullptr);
        if (p.q) {                                           // multinomial's check on the probabilities it samples
#pragma unroll
            for (int k = 0; k < PH_SLOTS; ++k)
                if (lane + 32 * k < A) bad |= !(fabsf(v[k]) < INFINITY);
        }
        bad = __any_sync(0xffffffffu, bad);
        float bv = -INFINITY;
        int bi = INT_MAX;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) {
            const int a = lane + 32 * k;
            if (a < A) {
                const float c = p.q ? v[k] / __ldg(p.q + (long long)n * A + a) : v[k];
                if (ph_better(c, a, bv, bi)) { bv = c; bi = a; }
            }
        }
#pragma unroll
        for (int s2 = 16; s2 >= 1; s2 >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, s2);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, s2);
            if (ph_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
        }
        if (p.probs) {
#pragma unroll
            for (int k = 0; k < PH_SLOTS; ++k) {
                const int a = lane + 32 * k;
                if (a < A) p.probs[(long long)n * A + a] = bad ? NAN : v[k];
            }
        }
        if (p.masked) {
#pragma unroll
            for (int k = 0; k < PH_SLOTS; ++k)
                if (lane + 32 * k < A) zs[warp][lane + 32 * k] = v[k];
        }
        __syncwarp();
        if (lane == 0) {
            float lp = zs[warp][bi];
            if (p.masked) lp = logf(fminf(fmaxf(lp, FLT_EPSILON), 1.f - FLT_EPSILON));   // probs_to_logits' clamp
            p.value[n] = bad ? NAN : zs[warp][A];
            p.action[n] = bad ? -1 : bi;
            p.log_prob[n] = bad ? NAN : lp;
            if (bad) atomicAdd(&refused, 1);
        }
    }
    __syncthreads();
    ph_publish(refused, p.ticket, p.status);
}

// The Linear stage of both head kernels: the CTA's ne feature rows from e0 into xs, then zs[e][r] = W_r . x_e + b_r
// for rows r < A of the actor and r = A the critic.  Warp w computes rows w, w + PH_WARPS, ...; ends synchronised.
__device__ __forceinline__ void ph_linear(const float* __restrict__ feat, const float* __restrict__ aw,
                                          const float* __restrict__ ab, const float* __restrict__ cw,
                                          const float* __restrict__ cb, int e0, int ne, int H, int A,
                                          float (*xs)[PH_MAX_H], float (*zs)[PH_MAX_A + 1]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < ne * H; i += 32 * PH_WARPS) xs[i / H][i % H] = __ldg(feat + (long long)e0 * H + i);
    __syncthreads();
    for (int r = warp; r <= A; r += PH_WARPS) {
        const float* __restrict__ w = r < A ? aw + (long long)r * H : cw;
        float acc[PH_ENVS];
#pragma unroll
        for (int e = 0; e < PH_ENVS; ++e) acc[e] = 0.f;
#pragma unroll 8
        for (int f = lane; f < H; f += 32) {
            const float wv = __ldg(w + f);
#pragma unroll
            for (int e = 0; e < PH_ENVS; ++e) acc[e] = fmaf(wv, xs[e][f], acc[e]);   // rows past ne: not stored
        }
        const float b = __ldg(r < A ? ab + r : cb);
#pragma unroll
        for (int e = 0; e < PH_ENVS; ++e) {
            const float s = ph_warp_sum(acc[e]);
            if (lane == 0 && e < ne) zs[e][r] = s + b;
        }
    }
    __syncthreads();
}

// The distribution stage of both head kernels, run by one warp on env n's logits z (shared, A values): lane l holds
// actions l + 32 k in v[k].  On return v holds the probabilities and, for the logits head, z the log-probabilities.
// Returns whether the reference's validated constructor refuses the row (lanes may disagree; callers vote).  save,
// when not NULL, receives what the training backward rebuilds the row from: the log-probabilities (masked = 0) or
// softmax(z) before the mask (masked = 1).
__device__ __forceinline__ bool ph_distribution(float* z, int masked, const float* __restrict__ mask, int n, int A,
                                                float (&v)[PH_SLOTS], float* save) {
    const int lane = threadIdx.x & 31;
    bool bad = false;
    float m = -INFINITY;
#pragma unroll
    for (int k = 0; k < PH_SLOTS; ++k) {
        const int a = lane + 32 * k;
        v[k] = a < A ? z[a] : -INFINITY;
        bad |= v[k] != v[k];
        m = fmaxf(m, v[k]);
    }
    m = ph_warp_max(m);
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < PH_SLOTS; ++k)
        if (lane + 32 * k < A) s += expf(v[k] - m);
    s = ph_warp_sum(s);
    if (!masked) {
        // logits = z - logsumexp(z), probs = softmax(logits); Categorical(logits=z) validates the normalised
        // logits, so a +Inf z (Inf - Inf) or an all -Inf row is refused like a NaN z
        const float lse = m + logf(s);
        float m2 = -INFINITY;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) {
            if (lane + 32 * k < A) {
                v[k] = v[k] - lse;
                bad |= v[k] != v[k];
            }
            m2 = fmaxf(m2, v[k]);
        }
        m2 = ph_warp_max(m2);
        float s2 = 0.f;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k)
            if (lane + 32 * k < A) s2 += expf(v[k] - m2);
        s2 = ph_warp_sum(s2);
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) {
            const int a = lane + 32 * k;
            if (a < A) {
                z[a] = v[k];                                 // log-probabilities, for the gather
                if (save) save[a] = v[k];
                v[k] = expf(v[k] - m2) / s2;
            }
        }
    } else {
        // probs = softmax(z) [* mask], then probs / probs.sum()
        float t = 0.f;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) {
            const int a = lane + 32 * k;
            if (a < A) {
                v[k] = expf(v[k] - m) / s;
                if (save) save[a] = v[k];
                if (mask) v[k] = __fmul_rn(v[k], __ldg(mask + (long long)n * A + a));   // rounded, then summed
                t += v[k];
            }
        }
        t = ph_warp_sum(t);
        bad |= t == 0.f;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k)
            if (lane + 32 * k < A) {
                v[k] = v[k] / t;
                bad |= !(v[k] >= 0.f);                   // NaN or negative
            }
    }
    return bad;
}

// ---------------------------------------------------------------------------
// The same heads in PPO's update, Policy.evaluate_actions after self.net (ss_baselines/av_nav/ppo/policy.py:70-82,
// savi :73-93, av_wan :68-80): value, log_probs(action) and the per-row entropy() for given actions, and their
// backward.  The forward runs policy_head_kernel's ph_linear and ph_distribution, so value and log_prob are the
// rollout's bits for the same features, weights and action.  The entropy is torch's -(clamp(logits, finfo.min) *
// probs).sum(-1), with the masked head's logits log(clamp_probs(p)).
// ---------------------------------------------------------------------------
struct PolicyHeadTrainParams {
    const float* feat;                 // [B][H]
    const float* aw;                   // [A][H]
    const float* ab;                   // [A]
    const float* cw;                   // [H]
    const float* cb;                   // [1]
    const float* mask;                 // [B][A] or NULL
    const long long* action;           // [B]
    float* value;                      // [B]
    float* log_prob;                   // [B]
    float* entropy;                    // [B]
    float* saved;                      // [B][A]: ph_distribution's save
    int* status;
    int* ticket;
    int B, H, A, masked;
};

// grid ceil(B / PH_ENVS), block 32 PH_WARPS
__global__ void __launch_bounds__(32 * PH_WARPS) policy_head_train_kernel(PolicyHeadTrainParams p) {
    __shared__ float xs[PH_ENVS][PH_MAX_H];
    __shared__ float zs[PH_ENVS][PH_MAX_A + 1];
    __shared__ int refused;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int e0 = blockIdx.x * PH_ENVS, ne = min(PH_ENVS, p.B - e0), A = p.A;
    if (threadIdx.x == 0) refused = 0;
    ph_linear(p.feat, p.aw, p.ab, p.cw, p.cb, e0, ne, p.H, A, xs, zs);
    if (warp < ne) {
        const int n = e0 + warp;
        float* z = zs[warp];
        float v[PH_SLOTS];
        const long long act = __ldg(p.action + n);
        const bool bad = __any_sync(0xffffffffu, ph_distribution(z, p.masked, p.mask, n, A, v, p.saved +
                                                                 (long long)n * A) || act < 0 || act >= A);
        float h = 0.f;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) {
            const int a = lane + 32 * k;
            if (a < A) {
                const float l = p.masked ? logf(fminf(fmaxf(v[k], FLT_EPSILON), 1.f - FLT_EPSILON))
                                         : fmaxf(z[a], -FLT_MAX);
                h = fmaf(l, v[k], h);
                if (p.masked) z[a] = v[k];
            }
        }
        h = ph_warp_sum(h);
        __syncwarp();
        if (lane == 0) {
            float lp = NAN;
            if (!bad) {
                lp = z[act];
                if (p.masked) lp = logf(fminf(fmaxf(lp, FLT_EPSILON), 1.f - FLT_EPSILON));
            }
            p.value[n] = bad ? NAN : z[A];
            p.log_prob[n] = lp;
            p.entropy[n] = bad ? NAN : -h;
            if (bad) atomicAdd(&refused, 1);
        }
    }
    __syncthreads();
    ph_publish(refused, p.ticket, p.status);
}

// Backward.  Kernel 1 (policy_head_dz_kernel): warp w of a CTA takes row n = PH_WARPS blockIdx.x + w, rebuilds its
// distribution from the saved row in the forward's order and writes dz = d(loss)/dz over the actor's A outputs; the CTA
// then forms dx = dz Wa + g_value Wc for its rows, each column summing actions in increasing order.  Kernel 2
// (policy_head_dw_kernel): the weight and bias gradients as one (A + 1) x (H + 1) matrix G = [dz | g_value]^T [x | 1],
// in 32 x 32 tiles; split s of PHW_SPLITS(B) sums its rows in increasing order, and the last split to finish a tile
// adds the splits' partial sums in split order.  No float atomics.
#define PHW_TILE 32
#define PHW_SPLIT_ROWS 128
#define PHW_MAX_SPLITS 64
#define PH_TRAIN_MAX_B SSB_POLICY_HEAD_TRAIN_MAX_B

static int phw_splits(int B) { return std::max(1, std::min((B + PHW_SPLIT_ROWS - 1) / PHW_SPLIT_ROWS, PHW_MAX_SPLITS)); }

struct PolicyHeadBackParams {
    const float* feat;                 // [B][H]
    const float* aw;                   // [A][H]
    const float* cw;                   // [H]
    const float* mask;                 // [B][A] or NULL
    const long long* action;           // [B]
    const float* saved;                // [B][A]
    const float* gv;                   // [B] upstream gradients of value, log_prob and entropy
    const float* glp;
    const float* gh;
    float* dz;                         // [B][A] workspace, NULL: no parameter gradient requested
    float* partial;                    // [splits][A + 1][H + 1] workspace
    int* tickets;                      // [tiles] workspace, zeroed by kernel 1
    float* dx;                         // [B][H] or NULL
    float* dwa;                        // [A][H] or NULL
    float* dba;                        // [A] or NULL
    float* dwc;                        // [H] or NULL
    float* dbc;                        // [1] or NULL
    int B, H, A, masked, splits, tiles;
};

// torch's autograd of value, log_probs(action) and entropy() for row n, one warp: d[k] = d(loss)/dz[lane + 32 k]
__device__ __forceinline__ void ph_row_backward(const PolicyHeadBackParams& p, int n, float (&d)[PH_SLOTS]) {
    const int lane = threadIdx.x & 31, A = p.A;
    const long long act = __ldg(p.action + n);
    const float glp = __ldg(p.glp + n), gh = __ldg(p.gh + n);
    const float* __restrict__ sv = p.saved + (long long)n * A;
    float x[PH_SLOTS], pr[PH_SLOTS];
    if (!p.masked) {
        // the saved log-probabilities l; probs = softmax(l) as the forward computed it
        float m2 = -INFINITY;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) {
            x[k] = lane + 32 * k < A ? __ldg(sv + lane + 32 * k) : -INFINITY;
            m2 = fmaxf(m2, x[k]);
        }
        m2 = ph_warp_max(m2);
        float s2 = 0.f;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k)
            if (lane + 32 * k < A) s2 += expf(x[k] - m2);
        s2 = ph_warp_sum(s2);
        // entropy = -sum(clamp(l, finfo.min) p): dp = -g clamp(l), dl = -g p where l >= finfo.min; softmax's
        // backward dl += p (dp - sum(p dp)); log_prob adds g to l[action]; logsumexp's dz = dl - exp(l) sum(dl)
        float sp = 0.f;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) {
            pr[k] = 0.f;
            d[k] = 0.f;
            if (lane + 32 * k < A) {
                pr[k] = expf(x[k] - m2) / s2;
                d[k] = -gh * fmaxf(x[k], -FLT_MAX);                   // dp
                sp = fmaf(pr[k], d[k], sp);
            }
        }
        sp = ph_warp_sum(sp);
        float sd = 0.f;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) {
            const int a = lane + 32 * k;
            if (a < A) {
                float dl = pr[k] * (d[k] - sp);
                if (x[k] >= -FLT_MAX) dl += -gh * pr[k];
                if (a == act) dl += glp;
                d[k] = dl;
                sd += dl;
            }
        }
        sd = ph_warp_sum(sd);
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k)
            if (lane + 32 * k < A) d[k] = fmaf(-expf(x[k]), sd, d[k]);
    } else {
        // the saved s = softmax(z); q = s [* mask] and t = sum(q) in the forward's order, P = q / t
        const float* __restrict__ mk = p.mask ? p.mask + (long long)n * A : nullptr;
        float t = 0.f;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) {
            const int a = lane + 32 * k;
            x[k] = 0.f;
            pr[k] = 0.f;
            if (a < A) {
                x[k] = __ldg(sv + a);
                pr[k] = mk ? __fmul_rn(x[k], __ldg(mk + a)) : x[k];
                t += pr[k];
            }
        }
        t = ph_warp_sum(t);
        // L = log(clamp(P, eps, 1 - eps)), entropy = -sum(L P): dL = -g P (+ g_lp at the action),
        // dP = -g L + dL / P where eps <= P <= 1 - eps; P = q / t: dq = dP / t - sum(dP P / t); ds = dq mask;
        // softmax's dz = s (ds - sum(s ds))
        float sdt = 0.f;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) {
            const int a = lane + 32 * k;
            d[k] = 0.f;
            if (a < A) {
                const float P = pr[k] / t;
                const float L = logf(fminf(fmaxf(P, FLT_EPSILON), 1.f - FLT_EPSILON));
                float dL = -gh * P;
                if (a == act) dL += glp;
                float dP = -gh * L;
                if (P >= FLT_EPSILON && P <= 1.f - FLT_EPSILON) dP += dL / P;
                d[k] = dP;
                sdt = fmaf(-dP, P / t, sdt);
            }
        }
        sdt = ph_warp_sum(sdt);
        float sr = 0.f;
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) {
            const int a = lane + 32 * k;
            if (a < A) {
                float ds = d[k] / t + sdt;
                if (mk) ds *= __ldg(mk + a);
                d[k] = ds;
                sr = fmaf(x[k], ds, sr);
            }
        }
        sr = ph_warp_sum(sr);
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k)
            if (lane + 32 * k < A) d[k] = x[k] * (d[k] - sr);
    }
}

// grid ceil(B / PH_WARPS), block 32 PH_WARPS
__global__ void __launch_bounds__(32 * PH_WARPS) policy_head_dz_kernel(PolicyHeadBackParams p) {
    __shared__ float dzs[PH_WARPS][PH_MAX_A];
    __shared__ float gvs[PH_WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, A = p.A, H = p.H;
    const int n0 = blockIdx.x * PH_WARPS, ne = min(PH_WARPS, p.B - n0), n = n0 + warp;
    if (p.dz && blockIdx.x == 0)
        for (int i = threadIdx.x; i < p.tiles; i += 32 * PH_WARPS) p.tickets[i] = 0;
    float d[PH_SLOTS];
    if (warp < ne) {
        ph_row_backward(p, n, d);
    } else {
#pragma unroll
        for (int k = 0; k < PH_SLOTS; ++k) d[k] = 0.f;
    }
#pragma unroll
    for (int k = 0; k < PH_SLOTS; ++k) {
        const int a = lane + 32 * k;
        if (a < A) {
            dzs[warp][a] = d[k];
            if (p.dz && warp < ne) p.dz[(long long)n * A + a] = d[k];
        }
    }
    if (lane == 0) gvs[warp] = warp < ne ? __ldg(p.gv + n) : 0.f;
    if (!p.dx) return;
    __syncthreads();
    for (int h = threadIdx.x; h < H; h += 32 * PH_WARPS) {
        float acc[PH_WARPS];
#pragma unroll
        for (int e = 0; e < PH_WARPS; ++e) acc[e] = 0.f;
#pragma unroll 4
        for (int j = 0; j < A; ++j) {
            const float w = __ldg(p.aw + (long long)j * H + h);
#pragma unroll
            for (int e = 0; e < PH_WARPS; ++e) acc[e] = fmaf(dzs[e][j], w, acc[e]);
        }
        const float c = __ldg(p.cw + h);
#pragma unroll
        for (int e = 0; e < PH_WARPS; ++e)
            if (e < ne) p.dx[(long long)(n0 + e) * H + h] = fmaf(gvs[e], c, acc[e]);
    }
}

// grid (ceil((H + 1) / 32), ceil((A + 1) / 32), splits), block 256: thread (tx, ty) owns column tx of the tile and
// rows ty + 8 i, i < 4
__global__ void __launch_bounds__(256) policy_head_dw_kernel(PolicyHeadBackParams p) {
    __shared__ float xs[PHW_TILE][PHW_TILE + 1];
    __shared__ float gs[PHW_TILE][PHW_TILE + 1];
    __shared__ bool last;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, H = p.H, A = p.A;
    const int h0 = blockIdx.x * PHW_TILE, j0 = blockIdx.y * PHW_TILE, s = blockIdx.z;
    const int per = (p.B + p.splits - 1) / p.splits, lo = s * per, hi = min(p.B, lo + per);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int r0 = lo; r0 < hi; r0 += PHW_TILE) {
        const int nr = min(PHW_TILE, hi - r0);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int i = threadIdx.x + 256 * q, rr = i >> 5, c = i & 31, h = h0 + c, j = j0 + c;
            const long long n = r0 + rr;
            float xv = 0.f, gv = 0.f;
            if (rr < nr) {
                xv = h < H ? __ldg(p.feat + n * H + h) : h == H ? 1.f : 0.f;
                gv = j < A ? p.dz[n * A + j] : j == A ? __ldg(p.gv + n) : 0.f;
            }
            xs[rr][c] = xv;
            gs[rr][c] = gv;
        }
        __syncthreads();
        for (int rr = 0; rr < nr; ++rr) {
            const float xv = xs[rr][tx];
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] = fmaf(gs[rr][ty + 8 * q], xv, acc[q]);
        }
        __syncthreads();
    }
    const int h = h0 + tx;
    const long long plane = (long long)(A + 1) * (H + 1);
    if (h <= H) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int j = j0 + ty + 8 * q;
            if (j <= A) p.partial[s * plane + (long long)j * (H + 1) + h] = acc[q];
        }
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(&p.tickets[blockIdx.y * gridDim.x + blockIdx.x], 1) == p.splits - 1;
    __syncthreads();
    if (!last || h > H) return;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int j = j0 + ty + 8 * q;
        if (j > A) continue;
        float g = 0.f;
        for (int t = 0; t < p.splits; ++t) g += __ldcg(p.partial + t * plane + (long long)j * (H + 1) + h);
        float* out = j < A ? (h < H ? (p.dwa ? p.dwa + (long long)j * H + h : nullptr) : (p.dba ? p.dba + j : nullptr))
                           : (h < H ? (p.dwc ? p.dwc + h : nullptr) : p.dbc);
        if (out) *out = g;
    }
}

// ---------------------------------------------------------------------------
// PPO's rollout storage (ss_baselines/common/rollout_storage.py, savi/models/rollout_storage.py).  Copies are
// described by fields (include/ssb200.h, ssb_rollout_field) and go through one grid-stride loop over every field's
// destination in the widest unit (16, 8, 4, 2 or 1 bytes) that divides the field's pointers, strides and row size,
// so the copy does not care what the elements are (actions are int64).
#define RO_FIELDS SSB_ROLLOUT_MAX_FIELDS
#define RO_THREADS 256

struct RoField {
    const char* src;
    char* dst;
    long long row_bytes, t_stride, o_stride;
    long long units;            // outer * T * n_cols * row_bytes >> unit_log2
    int T, outer, unit_log2;
};

struct RoCopyParams {
    RoField f[RO_FIELDS];
    int n_fields, n_cols, has_cols;
    int cols[SSB_ROLLOUT_MAX_COLS];
};

struct RoMemParams {
    float* masks;
    const float* not_done;
    float* em_out;
    int* status;
    int N, total, capacity, idx, step;
};

template <class V>
__device__ __forceinline__ void ro_copy_units(const RoField& f, int n_cols, const int* cols, long long i, long long stride) {
    const long long per_row = f.row_bytes / (long long)sizeof(V);
    for (; i < f.units; i += stride) {
        const long long r = i / per_row;
        const long long k = i - r * per_row;
        const int j = (int)(r % n_cols);
        const long long ot = r / n_cols;
        const int t = (int)(ot % f.T);
        const int o = (int)(ot / f.T);
        const int e = cols ? cols[j] : j;
        const V* s = reinterpret_cast<const V*>(f.src + o * f.o_stride + t * f.t_stride + e * f.row_bytes) + k;
        reinterpret_cast<V*>(f.dst)[i] = *s;
    }
}

__device__ void ro_copy_fields(const RoCopyParams& p) {
    const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const int* cols = p.has_cols ? p.cols : nullptr;
    for (int q = 0; q < p.n_fields; ++q) {
        const RoField& f = p.f[q];
        switch (f.unit_log2) {
            case 4: ro_copy_units<int4>(f, p.n_cols, cols, i0, stride); break;
            case 3: ro_copy_units<long long>(f, p.n_cols, cols, i0, stride); break;
            case 2: ro_copy_units<int>(f, p.n_cols, cols, i0, stride); break;
            case 1: ro_copy_units<short>(f, p.n_cols, cols, i0, stride); break;
            default: ro_copy_units<char>(f, p.n_cols, cols, i0, stride); break;
        }
    }
}

// One insert: every field, and with a memory (m.masks != NULL) ExternalMemory.insert's mask update of env row
// blockIdx.x (savi/models/rollout_storage.py:367-377): sum, overflow clear, set, multiply, em_masks[step + 1].
__global__ void __launch_bounds__(RO_THREADS)
rollout_insert_kernel(const __grid_constant__ RoCopyParams p, const __grid_constant__ RoMemParams m) {
    ro_copy_fields(p);
    if (!m.masks || (int)blockIdx.x >= m.N) return;
    __shared__ float red[RO_THREADS];
    const int e = blockIdx.x, tid = threadIdx.x;
    float* row = m.masks + (long long)e * m.total;
    float s = 0.f;
    for (int c = tid; c < m.total; c += RO_THREADS) s = __fadd_rn(s, row[c]);
    red[tid] = s;
    __syncthreads();
    for (int w = RO_THREADS / 2; w > 0; w >>= 1) {
        if (tid < w) red[tid] = __fadd_rn(red[tid], red[tid + w]);
        __syncthreads();
    }
    const float sum = red[0];
    const bool overflow = sum == (float)m.capacity;
    if (tid == 0 && sum > (float)m.capacity) {
        atomicAdd(m.status, 1);
        if (m.status[1 + e] == 0) m.status[1 + e] = m.step + 1;
    }
    int clear = m.idx - m.capacity;
    if (clear < 0) clear += m.total;                   // Python's negative index
    const float nd = m.not_done[e];
    float* out = m.em_out ? m.em_out + (long long)e * m.total : nullptr;
    for (int c = tid; c < m.total; c += RO_THREADS) {
        float v = row[c];
        if (overflow && c == clear) v = 0.f;
        if (c == m.idx) v = 1.f;
        v = __fmul_rn(v, nd);
        row[c] = v;
        if (out) out[c] = v;
    }
}

// One minibatch of recurrent_generator, or after_update's copies into slot 0.
__global__ void __launch_bounds__(RO_THREADS) rollout_gather_kernel(const __grid_constant__ RoCopyParams p) {
    ro_copy_fields(p);
}

struct RoReturnsParams {
    const float* rewards;
    float* value_preds;
    float* returns;
    const float* masks;
    const float* next_value;
    float* adv;
    float gamma, gamma_tau;
    int N, S, T, scan, use_gae, normalize;
};

#define RR_THREADS 1024

// Block-wide float64 sum in a fixed order: thread tid's values in index order, then a fixed tree.
__device__ double rr_block_sum(double v, double* red) {
    red[threadIdx.x] = v;
    __syncthreads();
    for (int w = RR_THREADS / 2; w > 0; w >>= 1) {
        if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    const double s = red[0];
    __syncthreads();
    return s;
}

// compute_returns for every env (one thread per env, T steps back to front), then the advantages over S rows.
// Every float32 operation is rounded once (__fmul_rn / __fadd_rn, no contraction), as the eager ops are.
__global__ void __launch_bounds__(RR_THREADS) rollout_returns_kernel(const RoReturnsParams p) {
    __shared__ double red[RR_THREADS];
    const int N = p.N;
    if (p.scan) {
        for (int e = threadIdx.x; e < N; e += RR_THREADS) {
            const float nv = p.next_value[e];
            if (p.use_gae) {
                p.value_preds[(long long)p.T * N + e] = nv;
                float gae = 0.f, v1 = nv;
#pragma unroll 4
                for (int t = p.T - 1; t >= 0; --t) {
                    const long long i = (long long)t * N + e;
                    const float v = p.value_preds[i], m1 = p.masks[i + N], r = p.rewards[i];
                    const float delta = __fsub_rn(__fadd_rn(r, __fmul_rn(__fmul_rn(p.gamma, v1), m1)), v);
                    gae = __fadd_rn(delta, __fmul_rn(__fmul_rn(p.gamma_tau, m1), gae));
                    p.returns[i] = __fadd_rn(gae, v);
                    v1 = v;
                }
            } else {
                p.returns[(long long)p.T * N + e] = nv;
                float R = nv;
#pragma unroll 4
                for (int t = p.T - 1; t >= 0; --t) {
                    const long long i = (long long)t * N + e;
                    R = __fadd_rn(__fmul_rn(__fmul_rn(R, p.gamma), p.masks[i + N]), p.rewards[i]);
                    p.returns[i] = R;
                }
            }
        }
        __syncthreads();
    }
    if (!p.adv) return;
    const long long n = (long long)p.S * N;
    double s = 0.0;
    for (long long i = threadIdx.x; i < n; i += RR_THREADS) {
        const float a = __fsub_rn(p.returns[i], p.value_preds[i]);
        p.adv[i] = a;
        s += (double)a;
    }
    if (!p.normalize) return;
    const double mean = rr_block_sum(s, red) / (double)n;
    double ss = 0.0;
    for (long long i = threadIdx.x; i < n; i += RR_THREADS) {
        const double d = (double)p.adv[i] - mean;
        ss += d * d;
    }
    const double var = rr_block_sum(ss, red) / (double)(n - 1);
    const float mf = (float)mean, den = __fadd_rn((float)sqrt(var), 1e-5f);
    for (long long i = threadIdx.x; i < n; i += RR_THREADS) p.adv[i] = __fdiv_rn(__fsub_rn(p.adv[i], mf), den);
}

// ---------------------------------------------------------------------------
// SAVi belief update (ss_baselines/savi/models/belief_predictor.py:136-202): the per-env part of
// BeliefPredictor.update after the location predictor and the label classifier have run.  One warp per env.
// Float32 arithmetic in the reference's numpy order: every product and sum is rounded on its own (__fmul_rn /
// __fadd_rn, never contracted to an FMA) and sqrtf / sinf / cosf / atan2f are the full-precision versions.
// ---------------------------------------------------------------------------
#define BELIEF_MAX_ENVS 1024
#define BELIEF_LABELS 21
#define BELIEF_WARPS 4

struct BeliefParams {
    const float* spec;                 // [B][spec_len]
    long long spec_len;
    const float* pose;                 // [B][pose_stride]: x, y, heading
    long long pose_stride;
    const float* loc_pred;             // [B][loc_stride], columns 0 and 1; NULL: no location belief
    long long loc_stride;
    const float* label_pred;           // [B][label_stride], columns 0..20; NULL: no label belief
    long long label_stride;
    float* last_pg;                    // [num_env][2] state in odometry coordinates
    unsigned char* loc_valid;          // [num_env]
    float* last_label;                 // [num_env][21]
    unsigned char* label_valid;        // [num_env]
    float* loc_out;                    // [B][2]
    float* cat_out;                    // [B][21]
    float w1, w;                       // float32(1 - w), float32(w)
    int current_pred_only;
    int B;
    unsigned int dones[BELIEF_MAX_ENVS / 32];
};

// Does the row hold any element != 0?  Scalar head up to 16-byte alignment, float4 body, scalar tail; the warp stops
// at the first chunk with a non-zero element.  NaN != 0, so NaN and Inf rows count as sounding, like sum() != 0.
__device__ __forceinline__ bool belief_row_nonzero(const float* __restrict__ row, long long n, int lane) {
    long long head = (long long)(((16u - ((unsigned)(uintptr_t)row & 15u)) & 15u) >> 2);
    if (head > n) head = n;
    const long long nv = (n - head) >> 2, tail0 = head + 4 * nv;
    bool nz = (lane < head && row[lane] != 0.f) || (lane < n - tail0 && row[tail0 + lane] != 0.f);
    if (__any_sync(0xffffffffu, nz)) return true;
    const float4* __restrict__ v = reinterpret_cast<const float4*>(row + head);
    for (long long c = 0; c < nv; c += 4 * 32) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const long long i = c + k * 32 + lane;
            if (i < nv) {
                const float4 x = __ldg(v + i);
                nz |= x.x != 0.f || x.y != 0.f || x.z != 0.f || x.w != 0.f;
            }
        }
        if (__any_sync(0xffffffffu, nz)) return true;
    }
    return false;
}

// odom_to_base (belief_predictor.py:219-226): delta = s - pose[:2]; theta = atan2(delta) - (-heading);
// d = |delta|; (d cos theta, d sin theta).
__device__ __forceinline__ float2 belief_odom_to_base(float sx, float sy, float px, float py, float angle) {
    const float dx = __fsub_rn(sx, px), dy = __fsub_rn(sy, py);
    const float th = __fsub_rn(atan2f(dy, dx), angle);
    const float d = sqrtf(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
    return make_float2(__fmul_rn(d, cosf(th)), __fmul_rn(d, sinf(th)));
}

// base_to_odom (belief_predictor.py:210-216): d = |a|; theta = atan2(a) + (-heading);
// (pose.x + d cos theta, pose.y + d sin theta).
__device__ __forceinline__ float2 belief_base_to_odom(float ax, float ay, float px, float py, float angle) {
    const float d = sqrtf(__fadd_rn(__fmul_rn(ax, ax), __fmul_rn(ay, ay)));
    const float th = __fadd_rn(atan2f(ay, ax), angle);
    return make_float2(__fadd_rn(px, __fmul_rn(d, cosf(th))), __fadd_rn(py, __fmul_rn(d, sinf(th))));
}

// grid ceil(B / BELIEF_WARPS), block 32 BELIEF_WARPS; warp = env.  Lanes 0..20 own one label column each, lane 0
// also the location.  State rows >= B are never touched.
__global__ void __launch_bounds__(32 * BELIEF_WARPS)
belief_update_kernel(const BeliefParams p) {
    const int lane = threadIdx.x & 31;
    const int env = blockIdx.x * BELIEF_WARPS + (threadIdx.x >> 5);
    if (env >= p.B) return;                                   // whole warps only: B is checked per warp
    const bool silent = !belief_row_nonzero(p.spec + (long long)env * p.spec_len, p.spec_len, lane);
    const bool done = (p.dones[env >> 5] >> (env & 31)) & 1u;
    const bool loc_valid = p.loc_pred && !done && p.loc_valid[env];
    const bool label_valid = p.label_pred && !done && p.label_valid[env];
    __syncwarp();                                              // every lane has read the flags before lane 0 writes them

    if (p.label_pred && lane < BELIEF_LABELS) {
        float* __restrict__ st = p.last_label + (long long)env * BELIEF_LABELS + lane;
        float avg;
        if (!silent) {
            const float l = __ldg(p.label_pred + (long long)env * p.label_stride + lane);
            avg = (!label_valid || p.current_pred_only) ? l : __fadd_rn(__fmul_rn(p.w1, l), __fmul_rn(p.w, *st));
            *st = avg;
        } else {
            avg = label_valid ? *st : (float)(1.0 / 21.0);        // np.ones(21) / 21 in float64, stored as float32
        }
        p.cat_out[(long long)env * BELIEF_LABELS + lane] = avg;
        if (lane == 0) p.label_valid[env] = (unsigned char)(label_valid || !silent);
    }

    if (p.loc_pred && lane == 0) {
        const float* __restrict__ ps = p.pose + (long long)env * p.pose_stride;
        const float px = __ldg(ps), py = __ldg(ps + 1), angle = -__ldg(ps + 2);
        float* __restrict__ st = p.last_pg + 2LL * env;
        float2 avg;
        if (!silent) {
            const float* __restrict__ pr = p.loc_pred + (long long)env * p.loc_stride;
            const float bx = -__ldg(pr + 1), by = __ldg(pr);
            if (!loc_valid || p.current_pred_only) {
                avg = make_float2(bx, by);
            } else {
                const float2 o = belief_odom_to_base(st[0], st[1], px, py, angle);
                avg = make_float2(__fadd_rn(__fmul_rn(p.w1, bx), __fmul_rn(p.w, o.x)),
                                  __fadd_rn(__fmul_rn(p.w1, by), __fmul_rn(p.w, o.y)));
            }
            const float2 s = belief_base_to_odom(avg.x, avg.y, px, py, angle);
            st[0] = s.x;
            st[1] = s.y;
        } else {
            avg = loc_valid ? belief_odom_to_base(st[0], st[1], px, py, angle) : make_float2(10.f, 10.f);
        }
        p.loc_out[2LL * env] = avg.x;
        p.loc_out[2LL * env + 1] = avg.y;
        p.loc_valid[env] = (unsigned char)(loc_valid || !silent);
    }
}

// ---------------------------------------------------------------------------
// SAVi's belief-predictor ResNet-18s (ssb_resnet18_batch, ssb_smt_resnet18_batch): one implicit-GEMM convolution
// kernel per conv (output channels x (env, pixel), K = IC KS KS split into a shape-fixed number of ranges), then one
// finish kernel per norm (sums the K ranges in order, BatchNorm from the live running statistics or GroupNorm over
// (env, group), residual, ReLU).  Every sum has a fixed order that depends on the layer's shape only, never on B.
// ---------------------------------------------------------------------------
#define RN_TK 16          // K rows per shared-memory tile
#define RN_THREADS 256    // 4 x 4 outputs per thread: TM x TN = 4096
#define RN_GROUPS 16      // finish kernel: CTAs per env (GroupNorm's 16 groups; BatchNorm uses the same split)
#define RN_MAX_ENVS 1024
#define RN_MAX_HW 256     // H, W limit of both entries
#define RN_CONVS 20       // stem + 8 blocks x 2 + 3 downsample convs, in module order
#define RN_MAX_IN 2       // networks of equal geometry one launch runs side by side (ssb_smt_cnn_batch: RGB, depth)

// The part of a conv that differs between the networks of one launch: parameters, activations and, for the stem,
// the input channels and hence the K split.
struct RnConvIn {
    const float* w;       // [OC][IC][KS][KS]
    const float* x;       // [B][IC][H][W], or the observation [B][H][W][2] (OBS)
    float* part;          // [S][B][OC][HO * WO] raw sums of K range s
    int IC, K, kps;       // kps: K rows per range, a multiple of RN_TK
};

struct RnConv {
    RnConvIn in[RN_MAX_IN];
    const float* labels;  // OBS: channel 2 + c reads labels[b * label_stride + c] inside the image, 0 in the padding
    long long label_stride;
    int B, H, W, OC, HO, WO, stride, pad, zs;   // zs: grid z slices per network (its largest K split)
};
static_assert(RN_MAX_IN == 2, "rn kernels select a network with one comparison");

template <int KS, bool OBS>
__device__ __forceinline__ float rn_tap(const RnConv& c, const RnConvIn& v, int b, int ih0, int iw0, int k, bool nvalid) {
    if (!nvalid || k >= v.K) return 0.f;
    const int ic = k / (KS * KS), r = k - ic * (KS * KS);
    const int ih = ih0 + r / KS, iw = iw0 + r % KS;
    if (ih < 0 || ih >= c.H || iw < 0 || iw >= c.W) return 0.f;
    if (OBS) {
        if (ic < 2) return __ldg(v.x + (((size_t)b * c.H + ih) * c.W + iw) * 2 + ic);
        return __ldg(c.labels + (size_t)b * c.label_stride + (ic - 2));
    }
    return __ldg(v.x + (((size_t)b * v.IC + ic) * c.H + ih) * c.W + iw);
}

// grid (ceil(B HO WO / TN), ceil(OC / TM), n_in zs): z = network i zs + K range s; slices past a network's own split
// exit.  Each output's sum runs over its K range in increasing k.
template <int KS, bool OBS, int TM>
__global__ void __launch_bounds__(RN_THREADS) rn_conv_kernel(const RnConv c) {
    static_assert(TM == 16 || TM == 32 || TM == 64, "tile");
    constexpr int TNN = 4096 / TM;                      // (env, pixel) columns per tile
    constexpr int A_PER = TM * RN_TK / RN_THREADS;      // weight tile loads per thread (1, 2, 4)
    constexpr int B_PER = TNN * RN_TK / RN_THREADS;     // input tile loads per thread (16, 8, 4)
    constexpr int B_KSTEP = RN_THREADS / TNN;
    __shared__ __align__(16) float As[RN_TK][TM];
    __shared__ __align__(16) float Bs[RN_TK][TNN];
    const int net = (int)blockIdx.z >= c.zs, s = (int)blockIdx.z - net * c.zs;
    const RnConvIn v = net ? c.in[1] : c.in[0];
    const int kb = s * v.kps;
    if (kb >= v.K) return;
    const int ke = min(v.K, kb + v.kps);
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * TM;
    const long long n0 = (long long)blockIdx.x * TNN;
    const int P = c.HO * c.WO;
    const long long N = (long long)c.B * P;
    // this thread's input column
    const long long nl = n0 + tid % TNN;
    const bool nvalid = nl < N;
    const int bl = nvalid ? (int)(nl / P) : 0, pl = nvalid ? (int)(nl - (long long)bl * P) : 0;
    const int ih0 = (pl / c.WO) * c.stride - c.pad, iw0 = (pl % c.WO) * c.stride - c.pad;
    const int bk = tid / TNN;
    // this thread's weight loads: row am, columns ak .. ak + A_PER - 1
    const int am = tid / (RN_TK / A_PER), ak = (tid % (RN_TK / A_PER)) * A_PER;
    const bool mvalid = m0 + am < c.OC;
    const float* wrow = v.w + (size_t)(mvalid ? m0 + am : 0) * v.K;
    float ra[A_PER], rb[B_PER];
    auto load = [&](int k0) {
#pragma unroll
        for (int j = 0; j < A_PER; ++j) {
            const int k = k0 + ak + j;
            ra[j] = (mvalid && k < ke) ? __ldg(wrow + k) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < B_PER; ++j) {
            const int k = k0 + bk + j * B_KSTEP;
            rb[j] = rn_tap<KS, OBS>(c, v, bl, ih0, iw0, k < ke ? k : v.K, nvalid);
        }
    };
    const int tm = tid / (TNN / 4), tn = tid % (TNN / 4);
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    load(kb);
    for (int k0 = kb; k0 < ke; k0 += RN_TK) {
#pragma unroll
        for (int j = 0; j < A_PER; ++j) As[ak + j][am] = ra[j];
#pragma unroll
        for (int j = 0; j < B_PER; ++j) Bs[bk + j * B_KSTEP][tid % TNN] = rb[j];
        __syncthreads();
        if (k0 + RN_TK < ke) load(k0 + RN_TK);
#pragma unroll
        for (int kk = 0; kk < RN_TK; ++kk) {
            const float4 a = *reinterpret_cast<const float4*>(&As[kk][tm * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tn * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
    float* part = v.part + (size_t)s * N * c.OC;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const long long n = n0 + tn * 4 + j;
        if (n >= N) continue;
        const int b = (int)(n / P), p = (int)(n - (long long)b * P);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int m = m0 + tm * 4 + i;
            if (m < c.OC) part[((size_t)b * c.OC + m) * P + p] = acc[i][j];
        }
    }
}

struct RnNorm {
    const float *gamma, *beta, *mean, *var;   // mean == NULL: GroupNorm over (env, group)
    float eps;
};

struct RnFinishIn {
    const float* a;      // [Sa][B][C][P] partial sums of the block's last conv (or the stem / a block's first conv)
    const float* d;      // [Sd][B][C][P] partial sums of the downsample conv, or NULL
    const float* r;      // [B][C][P] identity residual, or NULL
    float* out;          // [B][C][P]
    RnNorm na, nd;
    int Sa, Sd;
};

struct RnFinish {
    RnFinishIn in[RN_MAX_IN];
    int B, C, P, relu;
};

// Fixed-order sum over the 256 threads: xor tree in each warp, then the 8 warp sums in order.
__device__ __forceinline__ float rn_block_sum(float v, float* red) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < RN_THREADS / 32; ++w) t += red[w];
    __syncthreads();
    return t;
}

__device__ __forceinline__ float rn_parts(const float* p, int S, size_t stride, size_t i) {
    float v = p[i];
    for (int s = 1; s < S; ++s) v += p[s * stride + i];
    return v;
}

// GroupNorm statistics of one (env, group): biased variance, two passes.  Returns (mean, 1 / sqrt(var + eps)).
__device__ float2 rn_group_stats(const float* p, int S, size_t stride, size_t base, int E, float eps, float* red) {
    float s = 0.f;
    for (int e = threadIdx.x; e < E; e += RN_THREADS) s += rn_parts(p, S, stride, base + e);
    const float mean = rn_block_sum(s, red) / (float)E;
    float q = 0.f;
    for (int e = threadIdx.x; e < E; e += RN_THREADS) {
        const float v = rn_parts(p, S, stride, base + e) - mean;
        q = fmaf(v, v, q);
    }
    const float var = rn_block_sum(q, red) / (float)E;
    return make_float2(mean, 1.f / sqrtf(var + eps));
}

__device__ __forceinline__ float rn_norm(const RnNorm& n, float2 st, int c, float v) {
    if (n.mean) return (v - __ldg(n.mean + c)) * (__ldg(n.gamma + c) / sqrtf(__ldg(n.var + c) + n.eps)) + __ldg(n.beta + c);
    return (v - st.x) * st.y * __ldg(n.gamma + c) + __ldg(n.beta + c);
}

// grid (RN_GROUPS, B, n_in): channels [g C/16, (g+1) C/16) of env b of network z.
// out = act(norm_a(sum a) + (norm_d(sum d) | r | 0)).
__global__ void __launch_bounds__(RN_THREADS) rn_finish_kernel(const RnFinish p) {
    __shared__ float red[RN_THREADS / 32];
    const RnFinishIn f = blockIdx.z ? p.in[1] : p.in[0];
    const int g = blockIdx.x, b = blockIdx.y, Cg = p.C / RN_GROUPS, E = Cg * p.P;
    const size_t stride = (size_t)p.B * p.C * p.P, base = ((size_t)b * p.C + (size_t)g * Cg) * p.P;
    float2 sa = make_float2(0.f, 0.f), sd = sa;
    if (!f.na.mean) sa = rn_group_stats(f.a, f.Sa, stride, base, E, f.na.eps, red);
    if (f.d && !f.nd.mean) sd = rn_group_stats(f.d, f.Sd, stride, base, E, f.nd.eps, red);
    for (int e = threadIdx.x; e < E; e += RN_THREADS) {
        const int c = g * Cg + e / p.P;
        float v = rn_norm(f.na, sa, c, rn_parts(f.a, f.Sa, stride, base + e));
        if (f.d) v += rn_norm(f.nd, sd, c, rn_parts(f.d, f.Sd, stride, base + e));
        else if (f.r) v += f.r[base + e];
        f.out[base + e] = p.relu ? fmaxf(v, 0.f) : v;
    }
}

// What rn_finish_save_kernel keeps for ssb_smt_resnet18_train_backward_batch: the summed pre-norm values and the
// GroupNorm statistics exactly as the finish used them.
struct RnSave {
    float *za, *zd;       // [B][C][P] sum a, sum d (zd unused without d)
    float2 *sa, *sd;      // [B][RN_GROUPS] (mean, 1 / sqrt(var + eps)) of a and d
};

// rn_finish_kernel for one GroupNorm network (the training forward), with the same arithmetic in the same order, that
// also stores the sums and statistics.  A separate kernel rather than a flag, so rn_finish_kernel's code stays as it is.
__global__ void __launch_bounds__(RN_THREADS) rn_finish_save_kernel(const RnFinish p, const RnSave s) {
    __shared__ float red[RN_THREADS / 32];
    const RnFinishIn f = p.in[0];
    const int g = blockIdx.x, b = blockIdx.y, Cg = p.C / RN_GROUPS, E = Cg * p.P;
    const size_t stride = (size_t)p.B * p.C * p.P, base = ((size_t)b * p.C + (size_t)g * Cg) * p.P;
    float2 sd = make_float2(0.f, 0.f);
    const float2 sa = rn_group_stats(f.a, f.Sa, stride, base, E, f.na.eps, red);
    if (f.d) sd = rn_group_stats(f.d, f.Sd, stride, base, E, f.nd.eps, red);
    if (threadIdx.x == 0) {
        s.sa[(size_t)b * RN_GROUPS + g] = sa;
        if (f.d) s.sd[(size_t)b * RN_GROUPS + g] = sd;
    }
    for (int e = threadIdx.x; e < E; e += RN_THREADS) {
        const int c = g * Cg + e / p.P;
        const float za = rn_parts(f.a, f.Sa, stride, base + e);
        s.za[base + e] = za;
        float v = rn_norm(f.na, sa, c, za);
        if (f.d) {
            const float zd = rn_parts(f.d, f.Sd, stride, base + e);
            s.zd[base + e] = zd;
            v += rn_norm(f.nd, sd, c, zd);
        } else if (f.r) {
            v += f.r[base + e];
        }
        f.out[base + e] = p.relu ? fmaxf(v, 0.f) : v;
    }
}

struct RnHeadIn {
    const float* x;       // [B][C][P] the last block's output
    const float* w;       // [n_out][F]
    const float* bias;    // [n_out] or NULL
    int n_out, col;       // writes out[b][col .. col + n_out)
};

struct RnHead {
    RnHeadIn in[RN_MAX_IN];
    float* out;           // [B][ld]
    int C, P, avg, ld;
};

// grid (B, n_in): features = the per-channel mean over P pixels (avg, C <= 512) or the flattened [C][P] activation of
// network y, then out[b][col + j] = bias[j] + sum_f W[j][f] feat[f], one warp per output in a fixed order.
__global__ void __launch_bounds__(RN_THREADS) rn_head_kernel(const RnHead h) {
    __shared__ float pooled[512];
    const RnHeadIn v = blockIdx.y ? h.in[1] : h.in[0];
    const int b = blockIdx.x, C = h.C, P = h.P, avg = h.avg, F = avg ? C : C * P, n_out = v.n_out;
    const float* __restrict__ w = v.w;
    const float* __restrict__ bias = v.bias;
    float* __restrict__ out = h.out + (size_t)b * h.ld + v.col;
    const float* xb = v.x + (size_t)b * C * P;
    if (avg) {
        for (int ch = threadIdx.x; ch < C; ch += RN_THREADS) {
            float s = 0.f;
            for (int p = 0; p < P; ++p) s += xb[(size_t)ch * P + p];
            pooled[ch] = s / (float)P;
        }
        __syncthreads();
    }
    const float* feat = avg ? pooled : xb;
    const int lane = threadIdx.x & 31;
    for (int j = threadIdx.x >> 5; j < n_out; j += RN_THREADS / 32) {
        const float* wj = w + (size_t)j * F;
        float s = 0.f;
        for (int f = lane; f < F; f += 32) s = fmaf(__ldg(wj + f), feat[f], s);
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) out[j] = bias ? s + __ldg(bias + j) : s;
    }
}

// ---------------------------------------------------------------------------
// The backward of the SMT ResNet-18 (ssb_smt_resnet18_train_backward_batch).  Rows whose upstream gradient is all
// zero contribute nothing, so the first launch lists the live rows in order (srn_live_kernel) and every later kernel
// works on that compacted list: gradient buffers hold row j of the list at index j, saved activations are read at
// row live[j], and CTAs past the device-side count exit.  Every sum over rows runs in live-list order, so a batch's
// gradients are bit-identical to those of the same batch with its silent rows removed.
//   srn_live_kernel        live-row list and count
//   srn_fc_dw_kernel       fc dW = g^T F and db, summed over the live rows in order
//   srn_fc_dx_kernel       dF = g W
//   srn_norm_bwd_kernel    ReLU gradient on the saved output, GroupNorm backward of the main (and downsample) branch per
//                          (row, group), per-row dgamma / dbeta partials, and the identity branch's gradient
//   srn_dw_kernel          conv dW as an implicit GEMM over (live row, output pixel), zero padding, one partial per
//                          chunk of srn rows; srn_dw_reduce_kernel adds the chunks in order
//   srn_dx_kernel          conv dX in gather form (zero padding, stride 1 or 2), plus the other branch's gradient
//   srn_tap_kernel, srn_label_dw_kernel   the stem's label-channel weight gradient from per-row tap sums
//   srn_gn_reduce_kernel   dgamma / dbeta of all 20 norms from the per-row partials, in row order
// ---------------------------------------------------------------------------
#define SRN_MAX_ENVS 65535    // ssb_smt_resnet18_train_*: rows per call (the finish and norm grids put rows in y)
#define SRN_CHUNK 8192        // dW: (row, pixel) pairs per partial sum, rounded to whole rows

__device__ __forceinline__ bool srn_row_live(const float* g, int r, int n_out, int ld) {
    for (int o = 0; o < n_out; ++o)
        if (g[(size_t)r * ld + o] != 0.f) return true;    // NaN != 0: a non-finite row stays live
    return false;
}

// one CTA of 1024 threads: thread t scans rows [t per, (t + 1) per), then an inclusive scan of the counts.  In this
// kernel and the two fc kernels, g has row stride ld >= n_out.
__global__ void __launch_bounds__(1024) srn_live_kernel(const float* __restrict__ g, int B, int n_out, int ld,
                                                        int* __restrict__ live, int* __restrict__ count) {
    __shared__ int sc[1024];
    const int per = (B + 1023) / 1024, r0 = threadIdx.x * per, r1 = min(B, r0 + per);
    int n = 0;
    for (int r = r0; r < r1; ++r) n += srn_row_live(g, r, n_out, ld);
    sc[threadIdx.x] = n;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const int v = threadIdx.x >= o ? sc[threadIdx.x - o] : 0;
        __syncthreads();
        sc[threadIdx.x] += v;
        __syncthreads();
    }
    int pos = sc[threadIdx.x] - n;
    for (int r = r0; r < r1; ++r)
        if (srn_row_live(g, r, n_out, ld)) live[pos++] = r;
    if (threadIdx.x == 1023) *count = sc[1023];
}

// grid (ceil(F / 256), n_out): dW[o][f] = sum_j g[live j][o] F[live j][f]; thread f = 0 also db[o] (either may be NULL)
__global__ void __launch_bounds__(256) srn_fc_dw_kernel(const float* __restrict__ g, const float* __restrict__ feat,
                                                        const int* __restrict__ live, const int* __restrict__ count,
                                                        int ld, int F, float* dw, float* db) {
    const int f = blockIdx.x * 256 + threadIdx.x, o = blockIdx.y, cnt = *count;
    if (f >= F) return;
    float s = 0.f, sb = 0.f;
    for (int j = 0; j < cnt; ++j) {
        const int r = live[j];
        const float gv = g[(size_t)r * ld + o];
        s = fmaf(gv, feat[(size_t)r * F + f], s);
        sb += gv;
    }
    if (dw) dw[(size_t)o * F + f] = s;
    if (db && f == 0) db[o] = sb;
}

// grid (ceil(F / 256), B): dF[j][f] = sum_o g[live j][o] W[o][f]
__global__ void __launch_bounds__(256) srn_fc_dx_kernel(const float* __restrict__ g, const float* __restrict__ w,
                                                        const int* __restrict__ live, const int* __restrict__ count,
                                                        int n_out, int ld, int F, float* __restrict__ dF) {
    const int f = blockIdx.x * 256 + threadIdx.x, j = blockIdx.y;
    if (j >= *count || f >= F) return;
    const int r = live[j];
    float s = 0.f;
    for (int o = 0; o < n_out; ++o) s = fmaf(g[(size_t)r * ld + o], __ldg(w + (size_t)o * F + f), s);
    dF[(size_t)j * F + f] = s;
}

struct SrnNormBranch {
    const float* z;       // [B][C][P] saved pre-norm sums
    const float2* st;     // [B][RN_GROUPS] saved (mean, rstd)
    const float* gamma;   // [C]
    float* dz;            // [count][C][P] gradient of the pre-norm sums
    int col;              // first column of this norm's dgamma partials in a gpart row; dbeta follows at col + C
};

struct SrnNormBwd {
    const float* gin;     // [count][C][P] gradient of the finish output
    const float* y;       // [B][C][P] the finish output (after its ReLU)
    float* ds;            // [count][C][P] the ReLU's gradient, which the identity residual passes on, or NULL
    float* gpart;         // [count][CT] per-row dgamma / dbeta partials
    SrnNormBranch a, d;   // d.z NULL: no downsample branch
    const int *live, *count;
    int C, P, CT;
};

// grid (RN_GROUPS, B): row j of the list, group g.  dS = gin where y > 0 (threshold_backward), then for each branch
// x^ = (z - mean) rstd, dbeta_c = sum_p dS, dgamma_c = sum_p dS x^, and dz = rstd (gamma_c dS - (A + x^ Bs) / E) with
// A = sum_c gamma_c dbeta_c and Bs = sum_c gamma_c dgamma_c over the group's channels, every sum in a fixed order.
__global__ void __launch_bounds__(RN_THREADS) srn_norm_bwd_kernel(const SrnNormBwd p) {
    __shared__ float red[RN_THREADS / 32];
    __shared__ float sums[2][2][128 / RN_GROUPS];   // [branch][beta, gamma][channel of the group]; C <= 128
    const int g = blockIdx.x, j = blockIdx.y;
    if (j >= *p.count) return;
    const int r = p.live[j], Cg = p.C / RN_GROUPS, P = p.P, E = Cg * P;
    const size_t cj = ((size_t)j * p.C + (size_t)g * Cg) * P, cr = ((size_t)r * p.C + (size_t)g * Cg) * P;
    const int nb = p.d.z ? 2 : 1;
    for (int br = 0; br < nb; ++br) {
        const SrnNormBranch& q = br ? p.d : p.a;
        const float2 st = q.st[(size_t)r * RN_GROUPS + g];
        for (int cc = 0; cc < Cg; ++cc) {
            float sb = 0.f, sg = 0.f;
            for (int e = cc * P + threadIdx.x; e < (cc + 1) * P; e += RN_THREADS) {
                const float ds = p.y[cr + e] > 0.f ? p.gin[cj + e] : 0.f;
                sb += ds;
                sg = fmaf(ds, (q.z[cr + e] - st.x) * st.y, sg);
            }
            sb = rn_block_sum(sb, red);
            sg = rn_block_sum(sg, red);
            if (threadIdx.x == 0) {
                sums[br][0][cc] = sb;
                sums[br][1][cc] = sg;
                const size_t row = (size_t)j * p.CT + q.col + g * Cg + cc;
                p.gpart[row] = sg;
                p.gpart[row + p.C] = sb;
            }
        }
    }
    __syncthreads();
    float A[2], Bs[2];
    for (int br = 0; br < nb; ++br) {
        const SrnNormBranch& q = br ? p.d : p.a;
        A[br] = 0.f, Bs[br] = 0.f;
        for (int cc = 0; cc < Cg; ++cc) {
            const float gm = __ldg(q.gamma + g * Cg + cc);
            A[br] = fmaf(gm, sums[br][0][cc], A[br]);
            Bs[br] = fmaf(gm, sums[br][1][cc], Bs[br]);
        }
    }
    const float inv = 1.f / (float)E;
    for (int e = threadIdx.x; e < E; e += RN_THREADS) {
        const float ds = p.y[cr + e] > 0.f ? p.gin[cj + e] : 0.f;
        if (p.ds) p.ds[cj + e] = ds;
        for (int br = 0; br < nb; ++br) {
            const SrnNormBranch& q = br ? p.d : p.a;
            const float2 st = q.st[(size_t)r * RN_GROUPS + g];
            const float xh = (q.z[cr + e] - st.x) * st.y;
            const float gm = __ldg(q.gamma + g * Cg + e / P);
            q.dz[cj + e] = st.y * (gm * ds - fmaf(xh, Bs[br], A[br]) * inv);
        }
    }
}

struct SrnConvB {
    const float* x;       // dW: the conv's input, [B][IC][H][W] at row live[j], or the observation [B][H][W][2] (OBS)
    const float* dz;      // [count][OC][HO][WO] gradient of the conv output
    const float* w;       // dX: [OC][IC][KS][KS]
    const float* add;     // dX: [count][IC][H][W] added to the sum, or NULL
    float* out;           // dW: [chunks][OC][K] partial sums; dX: [count][IC][H][W]
    const int *live, *count;
    int IC, OC, H, W, HO, WO, stride, pad, K, rc;   // K: weight columns (IC KS KS); rc: rows per dW chunk
};

// The two backward GEMMs share rn_conv_kernel's tiling: TM x (4096 / TM) outputs per CTA, 4 x 4 per thread, RN_TK
// reduction steps per shared-memory tile, the next tile's loads in registers while the current one is multiplied.
template <int TM, class LoadA, class LoadB>
__device__ __forceinline__ void srn_gemm_tile(int kb, int ke, LoadA load_a, LoadB load_b, float (&acc)[4][4]) {
    constexpr int TNN = 4096 / TM, A_PER = TM * RN_TK / RN_THREADS, B_PER = TNN * RN_TK / RN_THREADS;
    constexpr int B_KSTEP = RN_THREADS / TNN;
    __shared__ __align__(16) float As[RN_TK][TM];
    __shared__ __align__(16) float Bs[RN_TK][TNN];
    const int tid = threadIdx.x, bk = tid / TNN;
    const int am = tid / (RN_TK / A_PER), ak = (tid % (RN_TK / A_PER)) * A_PER;
    float ra[A_PER], rb[B_PER];
    auto load = [&](int k0) {
#pragma unroll
        for (int j = 0; j < A_PER; ++j) ra[j] = k0 + ak + j < ke ? load_a(am, k0 + ak + j) : 0.f;
#pragma unroll
        for (int j = 0; j < B_PER; ++j) {
            const int k = k0 + bk + j * B_KSTEP;
            rb[j] = k < ke ? load_b(k) : 0.f;
        }
    };
    const int tm = tid / (TNN / 4), tn = tid % (TNN / 4);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    load(kb);
    for (int k0 = kb; k0 < ke; k0 += RN_TK) {
#pragma unroll
        for (int j = 0; j < A_PER; ++j) As[ak + j][am] = ra[j];
#pragma unroll
        for (int j = 0; j < B_PER; ++j) Bs[bk + j * B_KSTEP][tid % TNN] = rb[j];
        __syncthreads();
        if (k0 + RN_TK < ke) load(k0 + RN_TK);
#pragma unroll
        for (int kk = 0; kk < RN_TK; ++kk) {
            const float4 a = *reinterpret_cast<const float4*>(&As[kk][tm * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tn * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
}

// grid (chunks, ceil(K / (4096 / TM)), ceil(OC / TM)): chunk blockIdx.x covers list rows [x rc, (x + 1) rc); its
// partial dW[oc][k] sums dz[j][oc][p] X[(j, p)][k] over the chunk's (row, pixel) pairs in increasing order.  Column k
// = (ic, kh, kw) reads input pixel (oh s - pad + kh, ow s - pad + kw), 0 outside the image.
template <int KS, bool OBS, int TM>
__global__ void __launch_bounds__(RN_THREADS) srn_dw_kernel(const SrnConvB c) {
    constexpr int TNN = 4096 / TM, KK = KS * KS;
    const int cnt = *c.count, j0 = blockIdx.x * c.rc;
    if (j0 >= cnt) return;
    const int P = c.HO * c.WO, R = (min(cnt, j0 + c.rc) - j0) * P;
    const int m0 = blockIdx.z * TM, n0 = blockIdx.y * TNN, tid = threadIdx.x;
    const int kcol = n0 + tid % TNN;
    const bool kvalid = kcol < c.K;
    const int ic = kvalid ? kcol / KK : 0, t = kcol - ic * KK, kh = t / KS, kw = t % KS;
    const size_t zrow = (size_t)c.OC * P;
    auto load_a = [&](int m, int q) -> float {
        if (m0 + m >= c.OC) return 0.f;
        const int jj = q / P;
        return c.dz[(size_t)(j0 + jj) * zrow + (size_t)(m0 + m) * P + (q - jj * P)];
    };
    auto load_b = [&](int q) -> float {
        if (!kvalid) return 0.f;
        const int jj = q / P, p = q - jj * P;
        const int ih = (p / c.WO) * c.stride - c.pad + kh, iw = (p % c.WO) * c.stride - c.pad + kw;
        if (ih < 0 || ih >= c.H || iw < 0 || iw >= c.W) return 0.f;
        const size_t r = (size_t)__ldg(c.live + j0 + jj);
        if (OBS) return __ldg(c.x + ((r * c.H + ih) * c.W + iw) * 2 + ic);
        return __ldg(c.x + ((r * c.IC + ic) * c.H + ih) * c.W + iw);
    };
    float acc[4][4];
    srn_gemm_tile<TM>(0, R, load_a, load_b, acc);
    const int tm = tid / (TNN / 4), tn = tid % (TNN / 4);
    float* out = c.out + (size_t)blockIdx.x * c.OC * c.K;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + tm * 4 + i;
        if (m >= c.OC) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = n0 + tn * 4 + j;
            if (k < c.K) out[(size_t)m * c.K + k] = acc[i][j];
        }
    }
}

// dW[oc][koff + k] (row stride Kw) = the chunk partials of rows [0, count) added in chunk order
__global__ void __launch_bounds__(256) srn_dw_reduce_kernel(const float* __restrict__ part, const int* __restrict__ count,
                                                            int rc, int OC, int K, int Kw, float* __restrict__ dw) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= OC * K) return;
    const int chunks = (*count + rc - 1) / rc;
    float s = 0.f;
    for (int ch = 0; ch < chunks; ++ch) s += part[(size_t)ch * OC * K + i];
    dw[(size_t)(i / K) * Kw + i % K] = s;
}

// grid (ceil(count_max H W / (4096 / TM)), ceil(IC / TM)): dX[j][ic][ih][iw] = sum over (oc, kh, kw) of
// W[oc][ic][kh][kw] dz[j][oc][oh][ow] with oh s = ih + pad - kh, ow s = iw + pad - kw (taps that land off the output
// grid read 0), in increasing (oc, kh, kw), then + add[j][ic][ih][iw].
template <int KS, int TM>
__global__ void __launch_bounds__(RN_THREADS) srn_dx_kernel(const SrnConvB c) {
    constexpr int TNN = 4096 / TM, KK = KS * KS;
    const int Q = c.H * c.W, P = c.HO * c.WO, tid = threadIdx.x;
    const long long N = (long long)*c.count * Q, n0 = (long long)blockIdx.x * TNN;
    if (n0 >= N) return;
    const int m0 = blockIdx.y * TM;
    const long long nl = n0 + tid % TNN;
    const bool nvalid = nl < N;
    const long long jl = nvalid ? nl / Q : 0;
    const int ql = (int)(nl - jl * Q), ih = ql / c.W, iw = ql % c.W;
    const float* dzr = c.dz + (size_t)jl * c.OC * P;
    auto load_a = [&](int m, int k) -> float {
        if (m0 + m >= c.IC) return 0.f;
        const int oc = k / KK;
        return __ldg(c.w + ((size_t)oc * c.IC + m0 + m) * KK + (k - oc * KK));
    };
    auto load_b = [&](int k) -> float {
        if (!nvalid) return 0.f;
        const int oc = k / KK, t = k - oc * KK;
        const int th = ih + c.pad - t / KS, tw = iw + c.pad - t % KS;
        if (th < 0 || tw < 0) return 0.f;
        const int oh = th / c.stride, ow = tw / c.stride;
        if (oh * c.stride != th || ow * c.stride != tw || oh >= c.HO || ow >= c.WO) return 0.f;
        return dzr[(size_t)oc * P + oh * c.WO + ow];
    };
    float acc[4][4];
    srn_gemm_tile<TM>(0, c.OC * KK, load_a, load_b, acc);
    const int tm = tid / (TNN / 4), tn = tid % (TNN / 4);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const long long n = n0 + tn * 4 + j;
        if (n >= N) continue;
        const long long jj = n / Q;
        const int q = (int)(n - jj * Q);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int m = m0 + tm * 4 + i;
            if (m >= c.IC) continue;
            const size_t o = ((size_t)jj * c.IC + m) * Q + q;
            c.out[o] = c.add ? acc[i][j] + c.add[o] : acc[i][j];
        }
    }
}

// grid (OC, B): the stem's (stride 1, padding 3, 7 x 7) tap sums S[j][oc][kh][kw] = sum of dz[j][oc] over the output
// pixels whose tap (kh, kw) lands inside the image: column sums over the valid output rows, then over valid columns.
__global__ void __launch_bounds__(256) srn_tap_kernel(const float* __restrict__ dz, const int* __restrict__ count,
                                                      int OC, int H, int W, float* __restrict__ S) {
    __shared__ float T[7][RN_MAX_HW];
    const int oc = blockIdx.x, j = blockIdx.y;
    if (j >= *count) return;
    const float* g = dz + ((size_t)j * OC + oc) * H * W;
    for (int i = threadIdx.x; i < 7 * W; i += 256) {
        const int kh = i / W, ow = i % W, lo = max(0, 3 - kh), hi = min(H, H + 3 - kh);
        float s = 0.f;
        for (int oh = lo; oh < hi; ++oh) s += g[oh * W + ow];
        T[kh][ow] = s;
    }
    __syncthreads();
    if (threadIdx.x < 49) {
        const int kh = threadIdx.x / 7, kw = threadIdx.x % 7, lo = max(0, 3 - kw), hi = min(W, W + 3 - kw);
        float s = 0.f;
        for (int ow = lo; ow < hi; ++ow) s += T[kh][ow];
        S[((size_t)j * OC + oc) * 49 + threadIdx.x] = s;
    }
}

// dW[oc][2 + l][t] (row stride Kw) = sum_j labels[live j][l] S[j][oc][t], in list order
__global__ void __launch_bounds__(256) srn_label_dw_kernel(const float* __restrict__ labels, long long label_stride,
                                                           const float* __restrict__ S, const int* __restrict__ live,
                                                           const int* __restrict__ count, int OC, int NL, int Kw,
                                                           float* __restrict__ dw) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= OC * NL * 49) return;
    const int oc = i / (NL * 49), l = (i / 49) % NL, t = i % 49, cnt = *count;
    float s = 0.f;
    for (int j = 0; j < cnt; ++j)
        s = fmaf(__ldg(labels + (size_t)live[j] * label_stride + l), S[((size_t)j * OC + oc) * 49 + t], s);
    dw[(size_t)oc * Kw + (2 + l) * 49 + t] = s;
}

struct SrnGnOut {
    float* dgamma[RN_CONVS];
    float* dbeta[RN_CONVS];
    int C[RN_CONVS], col[RN_CONVS];
};

// grid (1, RN_CONVS): norm blockIdx.y, column c < C its dgamma, C <= c < 2C its dbeta; rows added in list order
__global__ void __launch_bounds__(256) srn_gn_reduce_kernel(const float* __restrict__ gpart, const int* __restrict__ count,
                                                            int CT, const SrnGnOut o) {
    const int n = blockIdx.y, C = o.C[n], cnt = *count;
    for (int c = threadIdx.x; c < 2 * C; c += 256) {
        float* dst = c < C ? o.dgamma[n] : o.dbeta[n];
        if (!dst) continue;
        float s = 0.f;
        for (int j = 0; j < cnt; ++j) s += gpart[(size_t)j * CT + o.col[n] + c];
        dst[c < C ? c : c - C] = s;
    }
}

// ---------------------------------------------------------------------------
// torchvision's ResNet-18 with BatchNorm in training or eval mode, forward and backward (ssb_resnet18_train_*: SAVi's
// AudioGoalPredictor pretraining).  The forward runs rn_conv_kernel, rn_finish_kernel, rn_head_kernel and, per norm:
//   brn_stats_kernel       conv i's K-range partials summed into z (kept for the backward) in rn_finish_kernel's order;
//                          training: per (chunk of rows, channel) FP64 sums of z - z0 and (z - z0)^2, z0 the channel's
//                          first value (the shift keeps E[z^2] - E[z]^2 from cancelling)
//   brn_update_kernel      training: per channel the batch mean and biased variance from the chunk sums in chunk order,
//                          running statistics and num_batches_tracked updated in place
//   rn_finish_kernel       on z (one K range) with the batch statistics, or the running ones in eval mode, as mean / var
//   brn_maxpool_kernel     the maxpool, with the window index of the element torch routes the gradient to
// The backward reuses the srn_* conv-gradient and fc-weight kernels on an identity row list (every row is live: under
// batch statistics a row with dy = 0 still gets dx != 0), and adds
//   brn_iota_kernel        that list
//   brn_pool_kernel        the avgpool features fc saw, rn_head_kernel's sums again
//   brn_fc_dx_kernel       dY = (g W) / (H4 W4) on every pixel of the last block: fc's and AdaptiveAvgPool2d's backward
//   brn_norm_sum_kernel    per (chunk, channel) FP64 sums of dS and dS x^ (dS: the ReLU gradient on the saved output)
//   brn_norm_total_kernel  per channel the chunk sums in order: dgamma, dbeta and the coefficients of dz
//   brn_norm_bwd_kernel    dz = gamma rstd (dS - sum dS / N - x^ sum dS x^ / N), the batch terms 0 in eval mode
//   brn_maxpool_bwd_kernel gather form over the windows that hold a pixel, in window order
// No float atomics anywhere: two runs give the same bits.
// ---------------------------------------------------------------------------
#define BRN_CHUNK 16384       // norm statistics: (row, pixel) pairs per chunk of one channel, rounded to whole rows

// rn_block_sum for N doubles at once
template <int N>
__device__ __forceinline__ void brn_block_sum(double (&v)[N], double (*red)[N]) {
#pragma unroll
    for (int k = 0; k < N; ++k)
#pragma unroll
        for (int o = 16; o; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int k = 0; k < N; ++k) red[threadIdx.x >> 5][k] = v[k];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < N; ++k) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < RN_THREADS / 32; ++w) t += red[w][k];
        v[k] = t;
    }
    __syncthreads();
}

struct BrnStats {
    const float* part;    // [S][B][C][P] partial sums of conv i
    float* z;             // [B][C][P]
    double2* sums;        // [chunks][C] (sum z - z0, sum (z - z0)^2), or NULL (eval mode: z only)
    int B, C, P, S, rc;   // rc: rows per chunk
};

// grid (C, chunks): channel blockIdx.x over rows [y rc, (y + 1) rc)
__global__ void __launch_bounds__(RN_THREADS) brn_stats_kernel(const BrnStats p) {
    __shared__ double red[RN_THREADS / 32][2];
    const int c = blockIdx.x, b0 = blockIdx.y * p.rc, n = (min(p.B, b0 + p.rc) - b0) * p.P;
    const size_t stride = (size_t)p.B * p.C * p.P;
    const double z0 = rn_parts(p.part, p.S, stride, (size_t)c * p.P);
    double v[2] = {0.0, 0.0};
    for (int e = threadIdx.x; e < n; e += RN_THREADS) {
        const size_t i = ((size_t)(b0 + e / p.P) * p.C + c) * p.P + e % p.P;
        const float z = rn_parts(p.part, p.S, stride, i);
        p.z[i] = z;
        const double d = (double)z - z0;
        v[0] += d;
        v[1] = fma(d, d, v[1]);
    }
    if (!p.sums) return;
    brn_block_sum<2>(v, red);
    if (threadIdx.x == 0) p.sums[(size_t)blockIdx.y * p.C + c] = make_double2(v[0], v[1]);
}

struct BrnUpdate {
    const double2* sums;  // brn_stats_kernel's chunk sums
    const float* z;       // z0 of channel c is z[c P]
    float *mean, *var;    // [C] batch mean and biased variance, what the finish normalises with
    double* dmean;        // [C] the batch mean in FP64, what the backward centres with
    float *run_mean, *run_var;
    int64_t* nbt;         // num_batches_tracked, or NULL
    long long N;          // B P values per channel, N >= 2
    int C, P, chunks;
    float momentum;
};

// grid ceil(C / 256): running = (1 - m) running + m batch, with the unbiased variance (N / (N - 1)) for running_var
__global__ void __launch_bounds__(256) brn_update_kernel(const BrnUpdate p) {
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (c == 0 && p.nbt) *p.nbt += 1;
    if (c >= p.C) return;
    double s = 0.0, q = 0.0;
    for (int k = 0; k < p.chunks; ++k) {
        const double2 v = p.sums[(size_t)k * p.C + c];
        s += v.x;
        q += v.y;
    }
    const double N = (double)p.N, m = s / N, var = fmax(q / N - m * m, 0.0), mean = (double)p.z[(size_t)c * p.P] + m;
    const double mo = (double)p.momentum;
    p.mean[c] = (float)mean;
    p.var[c] = (float)var;
    p.dmean[c] = mean;
    p.run_mean[c] = (float)((1.0 - mo) * (double)p.run_mean[c] + mo * mean);
    p.run_var[c] = (float)((1.0 - mo) * (double)p.run_var[c] + mo * var * N / (N - 1.0));
}

// torchvision's MaxPool2d(3, 2, 1): [B][C][H][W] -> [B][C][HO][WO], the padding never wins; unless arg is NULL, also
// the window index 3 dh + dw of the element torch's max_pool2d picks: the first maximum in row-major window order, a
// NaN taking the window
__global__ void brn_maxpool_kernel(const float* __restrict__ x, int BC, int H, int W, int HO, int WO,
                                   float* __restrict__ out, unsigned char* __restrict__ arg) {
    const long long n = (long long)BC * HO * WO;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int ow = (int)(i % WO), oh = (int)((i / WO) % HO);
        const long long bc = i / ((long long)HO * WO);
        const float* p = x + bc * H * W;
        float m = -INFINITY, t = -INFINITY;
        int a = -1;
        for (int dh = 0; dh < 3; ++dh) {
            const int ih = oh * 2 - 1 + dh;
            if (ih < 0 || ih >= H) continue;
            for (int dw = 0; dw < 3; ++dw) {
                const int iw = ow * 2 - 1 + dw;
                if (iw < 0 || iw >= W) continue;
                const float v = p[ih * W + iw];
                m = fmaxf(m, v);
                if (a < 0 || v > t || v != v) t = v, a = dh * 3 + dw;
            }
        }
        out[i] = m;
        if (arg) arg[i] = (unsigned char)a;
    }
}

// grid-stride over the stem output [B C][H][W]: dX = the sum of dY over the windows (oh, ow) that hold the pixel and
// picked it, in increasing (oh, ow)
__global__ void brn_maxpool_bwd_kernel(const float* __restrict__ dy, const unsigned char* __restrict__ arg, int BC,
                                       int H, int W, int HO, int WO, float* __restrict__ dx) {
    const long long n = (long long)BC * H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int iw = (int)(i % W), ih = (int)((i / W) % H);
        const long long o = i / ((long long)H * W) * HO * WO;
        float s = 0.f;
        for (int oh = ih / 2; oh <= min(HO - 1, (ih + 1) / 2); ++oh)
            for (int ow = iw / 2; ow <= min(WO - 1, (iw + 1) / 2); ++ow)
                if (arg[o + oh * WO + ow] == (ih - 2 * oh + 1) * 3 + (iw - 2 * ow + 1)) s += dy[o + oh * WO + ow];
        dx[i] = s;
    }
}

__global__ void brn_iota_kernel(int B, int* __restrict__ live) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= B; i += gridDim.x * blockDim.x) live[i] = i;   // live[B] = B: the count
}

// grid (B): feat[b][c] = rn_head_kernel's mean of x[b][c] over P pixels
__global__ void __launch_bounds__(RN_THREADS) brn_pool_kernel(const float* __restrict__ x, int C, int P,
                                                              float* __restrict__ feat) {
    const float* xb = x + (size_t)blockIdx.x * C * P;
    for (int ch = threadIdx.x; ch < C; ch += RN_THREADS) {
        float s = 0.f;
        for (int p = 0; p < P; ++p) s += xb[(size_t)ch * P + p];
        feat[(size_t)blockIdx.x * C + ch] = s / (float)P;
    }
}

// grid (ceil(C / 256), B): dY[b][c][p] = (sum_o g[b][o] W[o][c]) / P on every pixel p
__global__ void __launch_bounds__(256) brn_fc_dx_kernel(const float* __restrict__ g, const float* __restrict__ w,
                                                        int n_out, int C, int P, float* __restrict__ dy) {
    const int c = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
    if (c >= C) return;
    float s = 0.f;
    for (int o = 0; o < n_out; ++o) s = fmaf(g[(size_t)b * n_out + o], __ldg(w + (size_t)o * C + c), s);
    const float v = s / (float)P;
    for (int p = 0; p < P; ++p) dy[((size_t)b * C + c) * P + p] = v;
}

struct BrnBranch {
    const float* z;           // [B][C][P] saved pre-norm sums
    const float *mean, *var;  // [C] what the forward normalised with: the batch statistics, or the running ones (eval)
    const double* dmean;      // [C] training: the batch mean in FP64, so that x^ and with it dz sum to 0 over the
                              // channel as exactly as FP64 allows
    const float* gamma;
    double2* sums;            // [chunks][C] (sum dS, sum dS x^)
    double4* coef;            // [C] (gamma rstd, sum dS / N, sum dS x^ / N, rstd); the middle two 0 in eval mode
    float* dz;                // [B][C][P]
    float *dgamma, *dbeta;    // [C] or NULL
    float eps;
};

struct BrnNormBwd {
    const float* gin;     // [B][C][P] gradient of the finish output
    const float* y;       // [B][C][P] the finish output (after its ReLU)
    float* ds;            // the ReLU gradient, which the identity residual passes on, or NULL
    BrnBranch a, d;       // d.z NULL: no downsample branch
    int B, C, P, rc, chunks, training;
};

__device__ __forceinline__ float brn_rstd(const BrnBranch& q, int c) { return 1.f / sqrtf(__ldg(q.var + c) + q.eps); }

__device__ __forceinline__ double brn_mean(const BrnBranch& q, int c) {
    return q.dmean ? q.dmean[c] : (double)__ldg(q.mean + c);
}

// grid (C, chunks) as brn_stats_kernel
__global__ void __launch_bounds__(RN_THREADS) brn_norm_sum_kernel(const BrnNormBwd p) {
    __shared__ double red[RN_THREADS / 32][3];
    const int c = blockIdx.x, b0 = blockIdx.y * p.rc, n = (min(p.B, b0 + p.rc) - b0) * p.P;
    const bool two = p.d.z != nullptr;
    const double ma = brn_mean(p.a, c), ra = brn_rstd(p.a, c);
    const double md = two ? brn_mean(p.d, c) : 0.0, rd = two ? brn_rstd(p.d, c) : 0.0;
    double v[3] = {0.0, 0.0, 0.0};
    for (int e = threadIdx.x; e < n; e += RN_THREADS) {
        const size_t i = ((size_t)(b0 + e / p.P) * p.C + c) * p.P + e % p.P;
        const float ds = p.y[i] > 0.f ? p.gin[i] : 0.f;
        v[0] += ds;
        v[1] = fma((double)ds, ((double)p.a.z[i] - ma) * ra, v[1]);
        if (two) v[2] = fma((double)ds, ((double)p.d.z[i] - md) * rd, v[2]);
    }
    brn_block_sum<3>(v, red);
    if (threadIdx.x == 0) {
        const size_t k = (size_t)blockIdx.y * p.C + c;
        p.a.sums[k] = make_double2(v[0], v[1]);
        if (two) p.d.sums[k] = make_double2(v[0], v[2]);
    }
}

// grid (ceil(C / 256), branches)
__global__ void __launch_bounds__(256) brn_norm_total_kernel(const BrnNormBwd p) {
    const int c = blockIdx.x * 256 + threadIdx.x;
    const BrnBranch& q = blockIdx.y ? p.d : p.a;
    if (c >= p.C) return;
    double sb = 0.0, sg = 0.0;
    for (int k = 0; k < p.chunks; ++k) {
        const double2 v = q.sums[(size_t)k * p.C + c];
        sb += v.x;
        sg += v.y;
    }
    if (q.dgamma) q.dgamma[c] = (float)sg;
    if (q.dbeta) q.dbeta[c] = (float)sb;
    const double N = (double)p.B * p.P, r = brn_rstd(q, c);
    q.coef[c] = make_double4((double)__ldg(q.gamma + c) * r, p.training ? sb / N : 0.0, p.training ? sg / N : 0.0, r);
}

// grid (C, chunks) as brn_norm_sum_kernel
__global__ void __launch_bounds__(RN_THREADS) brn_norm_bwd_kernel(const BrnNormBwd p) {
    const int c = blockIdx.x, b0 = blockIdx.y * p.rc, n = (min(p.B, b0 + p.rc) - b0) * p.P;
    const bool two = p.d.z != nullptr;
    const double4 ka = p.a.coef[c], kd = two ? p.d.coef[c] : make_double4(0.0, 0.0, 0.0, 0.0);
    const double ma = brn_mean(p.a, c), md = two ? brn_mean(p.d, c) : 0.0;
    for (int e = threadIdx.x; e < n; e += RN_THREADS) {
        const size_t i = ((size_t)(b0 + e / p.P) * p.C + c) * p.P + e % p.P;
        const float ds = p.y[i] > 0.f ? p.gin[i] : 0.f;
        if (p.ds) p.ds[i] = ds;
        p.a.dz[i] = (float)(ka.x * ((double)ds - ka.y - ((double)p.a.z[i] - ma) * ka.w * ka.z));
        if (two) p.d.dz[i] = (float)(kd.x * ((double)ds - kd.y - ((double)p.d.z[i] - md) * kd.w * kd.z));
    }
}

// SMTCNN's input stage (ssb_smt_cnn_batch): permute, optional / 255, the area resize of ResizeCenterCropper and its
// centre crop, into the [B][C][64][64] image the stem reads.  Crop pixel (y, x) is resized pixel (Y, X) = (y + cy,
// x + cx), the mean of input rows [Y H / rh, ceil((Y + 1) H / rh)) and columns [X W / rw, ceil((X + 1) W / rw)),
// summed row by row in increasing order and divided by the bin's height, then by its width (adaptive_avg_pool2d).
// Each scaled value is rounded to float32 before it is added (__fmul_rn keeps nvcc from contracting the multiply
// into the sum's FFMA), as the reference materialises x / 255 before it resizes.
#define CNN_CROP 64
#define CNN_TRAIN_GRADS (3 * RN_CONVS + 2)   // ssb_smt_cnn_train_backward_batch: gradient pointers per input

struct CnnPrepIn {
    const float* obs;     // [B][H][W][C]
    float* img;           // [B][C][64][64]
    float mul;            // 1 / 255 or 1, applied to every loaded value
    int C, H, W, rh, rw, cy, cx;
};

struct CnnPrep {
    CnnPrepIn in[RN_MAX_IN];
    int B;
};

// grid (64 * 64 / 256, B, n_in): one crop pixel of one env per thread, every channel
__global__ void __launch_bounds__(256) cnn_prep_kernel(const CnnPrep p) {
    const CnnPrepIn v = blockIdx.z ? p.in[1] : p.in[0];
    const int px = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
    const int Y = px / CNN_CROP + v.cy, X = px % CNN_CROP + v.cx;
    const int h0 = Y * v.H / v.rh, h1 = ((Y + 1) * v.H + v.rh - 1) / v.rh;
    const int w0 = X * v.W / v.rw, w1 = ((X + 1) * v.W + v.rw - 1) / v.rw;
    const float* src = v.obs + (size_t)b * v.H * v.W * v.C;
    float* dst = v.img + (size_t)b * v.C * CNN_CROP * CNN_CROP + px;
    for (int c = 0; c < v.C; ++c) {
        float s = 0.f;
        for (int ih = h0; ih < h1; ++ih)
            for (int iw = w0; iw < w1; ++iw) s += __fmul_rn(__ldg(src + ((size_t)ih * v.W + iw) * v.C + c), v.mul);
        dst[(size_t)c * CNN_CROP * CNN_CROP] = s / (float)(h1 - h0) / (float)(w1 - w0);
    }
}

// ---------------------------------------------------------------------------
// SAVi's scene memory transformer (ssb_smt_state_encoder_batch): SMTStateEncoder.single_forward with one encoder and
// one decoder layer, on each env's valid tokens only.  Token rows are compacted per env: row j < cnt[b] of env b is
// its j-th valid memory slot in slot order, and row cnt[b] - 1 is the current observation.  Six launches:
//   smt_fuse_kernel     mask scan + compaction, pose encoding, pose_encoder, fusion_encoder (two chained linears)
//   smt_linear_kernel   the encoder's QKV projection, and later the decoder's cross-attention K/V projection
//   smt_attn_kernel     encoder self-attention per (env, head, 16 queries) over the env's valid keys
//   smt_enc_tail_kernel out_proj + residual + norm1, FF + residual + norm2, encoder.norm
//   smt_decoder_kernel  the whole decoder for SMT_DEC_ENVS envs per CTA (weights read once per CTA)
// Every sum runs in an order fixed by the layer's shape: GEMM K loops in increasing k, softmax max / sum and P.V in
// slot order, LayerNorm mean / variance over a fixed lane split.  None depends on B or on other envs, so an env's
// output is bit-identical at any B, at any position in the batch, and whatever its masked slots hold (never read).
// The row GEMMs keep their own tiling rather than rn_conv_kernel's: their epilogues need whole d-wide rows in one CTA
// (residual + LayerNorm), several GEMMs chain inside one kernel, and the rows are ragged per env (cnt on the device).
// ---------------------------------------------------------------------------
#define SMT_THREADS 256
#define SMT_RT 16            // token rows per CTA (fuse, linear, attention queries, encoder tail)
#define SMT_DEC_ENVS 4       // decoder: envs per CTA
#define SMT_WS 8256          // weight tile floats: KT x (NC + 1) with NC * KT = 8192
#define SMT_KT_KEYS 64       // attention: keys per shared-memory tile
#define SMT_MAX_ENVS 1024
#define SMT_MAX_TOKENS 1024  // M + 1
#define SMT_MAX_D 512
#define SMT_MAX_HD 128
#define SMT_MAX_IN 1024
// dynamic shared memory at the limits (bytes), opted into once per device in ssb_create
#define SMT_SMEM_FUSE ((SMT_RT * (SMT_MAX_IN + 16) + SMT_RT * SMT_MAX_D + SMT_WS + SMT_RT + 8) * 4)
#define SMT_SMEM_LIN ((SMT_RT * 3 * SMT_MAX_D + SMT_WS) * 4)   // K up to 3 d_model: the backward's dX of the QKV rows
#define SMT_SMEM_ATTN ((SMT_RT * SMT_MAX_HD + SMT_KT_KEYS * (SMT_MAX_HD + 1) + SMT_RT * SMT_MAX_TOKENS) * 4)
#define SMT_SMEM_TAIL ((3 * SMT_RT * SMT_MAX_D + SMT_WS) * 4)
#define SMT_SMEM_DEC ((4 * SMT_DEC_ENVS * SMT_MAX_D + 8 * SMT_MAX_TOKENS) * 4)

struct SmtLin { const float* w; const float* b; };
struct SmtLn { const float* g; const float* b; float eps; };

struct SmtArgs {
    const float* x;        // [B][d_in]
    const float* memory;   // [M][B][d_in]
    const float* masks;    // [B][M]
    const float* goal;     // [B][d] or NULL
    int* cnt;              // [B] valid tokens per env (current token included)
    float* h0;             // [B][T][d] fused tokens
    float* qkv;            // [B][T][3d] encoder QKV, then the decoder's cross-attention K / V ([B][T][2d] rows)
    float* att;            // [B][T][d] attention output
    float* enc;            // [B][T][d] encoder output E (the rollout: att, in place)
    float* kv;             // [B][T][2d] the decoder's cross-attention K / V rows (the rollout: qkv, in place)
    float* out;            // [B][d]
    // kept for ssb_smt_state_encoder_train_backward_batch; NULL at rollout
    int* slot;             // [B][T] memory slot of each compacted row (M: the current token)
    float* xin;            // [B][T][Fp] fusion_encoder[0]'s input rows
    float* hid;            // [B][T][d] fusion_encoder's hidden ReLU
    float* u;              // [B][T][2][d] the encoder tail's LayerNorm inputs (norm1, norm2)
    float* ffh;            // [B][T][d] the encoder FF's hidden ReLU
    float* st;             // [B][T][6] (mean, rstd) of norm1, norm2 and encoder.norm
    SmtLin pose, fuse1, fuse2, enc_qkv, enc_out, enc_ff1, enc_ff2, dec_v, dec_sa_out, dec_q, dec_kv, dec_ca_out,
        dec_ff1, dec_ff2;
    SmtLn enc_n1, enc_n2, enc_n, dec_n1, dec_n2, dec_n3, dec_n;
    int B, M, T, d_in, pi, F, d, H, hd, pretraining;
};

// out[r][n] = act(bias[n] + sum_k X[r][k] W[n][k]) for the RT rows of X (shared memory, row stride ldx) and n < N,
// k ascending in one fma chain per output.  Each thread owns TR rows x 4 columns (lane + 32 j) of a chunk of NC
// columns; the weight tile Ws[KT][NC + 1] is staged transposed.  Rows >= nrows are computed but not stored.
template <int RT, int TR>
__device__ void smt_block_linear(const float* X, int ldx, int K, const float* __restrict__ W,
                                 const float* __restrict__ bias, int N, float* Ws, float* dst, int ldd, int nrows,
                                 bool relu) {
    constexpr int RG = RT / TR, CG = 8 / RG, NC = CG * 128, KT = 8192 / NC, LDW = NC + 1;
    static_assert(RG * CG == 8 && KT * LDW <= SMT_WS, "tile");
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, rg = warp % RG, cg = warp / RG;
    constexpr int PER = NC * KT / SMT_THREADS;       // weight tile loads per thread, all in flight together
    float pre[PER];
    auto fetch = [&](int n0, int k0) {
        const int kn = min(KT, K - k0);
#pragma unroll
        for (int m = 0; m < PER; ++m) {
            const int i = threadIdx.x + m * SMT_THREADS, kk = i % KT, n = n0 + i / KT;
            pre[m] = (n < N && kk < kn) ? __ldg(W + (size_t)n * K + k0 + kk) : 0.f;
        }
    };
    fetch(0, 0);
    for (int n0 = 0; n0 < N; n0 += NC) {
        float acc[TR][4];
#pragma unroll
        for (int i = 0; i < TR; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
        for (int k0 = 0; k0 < K; k0 += KT) {
            const int kn = min(KT, K - k0);
#pragma unroll
            for (int m = 0; m < PER; ++m) {
                const int i = threadIdx.x + m * SMT_THREADS;
                Ws[(i % KT) * LDW + i / KT] = pre[m];
            }
            __syncthreads();
            if (k0 + KT < K) fetch(n0, k0 + KT);          // the next tile loads while this one is used
            else if (n0 + NC < N) fetch(n0 + NC, 0);
            const float* xr = X + (size_t)rg * TR * ldx + k0;
            const float* wc = Ws + cg * 128 + lane;
#pragma unroll 4
            for (int kk = 0; kk < kn; ++kk) {
                float a[TR], w[4];
#pragma unroll
                for (int i = 0; i < TR; ++i) a[i] = xr[i * ldx + kk];
#pragma unroll
                for (int j = 0; j < 4; ++j) w[j] = wc[kk * LDW + 32 * j];
#pragma unroll
                for (int i = 0; i < TR; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
            }
            __syncthreads();
        }
#pragma unroll
        for (int i = 0; i < TR; ++i) {
            const int r = rg * TR + i;
            if (r >= nrows) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int n = n0 + cg * 128 + lane + 32 * j;
                if (n >= N) continue;
                const float v = acc[i][j] + __ldg(bias + n);
                dst[(size_t)r * ldd + n] = relu ? fmaxf(v, 0.f) : v;
            }
        }
    }
}

// Fixed-order warp sum: lane-strided partial sums, then an xor tree (every lane ends with the same value).
__device__ __forceinline__ float smt_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float smt_warp_max(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// out[r][n] = act(bias[n] + sum_k X[r][k] W[n][k]) for R rows of X (shared memory, [R][K]) into dst ([R][N]): one warp
// per 4 outputs, lanes over k (coalesced weight rows, every weight read once per CTA), then a fixed-order warp sum.
template <int R>
__device__ void smt_rows_gemv(const float* X, int K, const float* __restrict__ W, const float* __restrict__ bias, int N,
                              float* dst, bool relu) {
    constexpr int G = 4;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int n0 = warp * G; n0 < N; n0 += (SMT_THREADS / 32) * G) {
        float acc[G][R];
#pragma unroll
        for (int g = 0; g < G; ++g)
#pragma unroll
            for (int r = 0; r < R; ++r) acc[g][r] = 0.f;
#pragma unroll 4
        for (int k = lane; k < K; k += 32) {
            float w[G];
#pragma unroll
            for (int g = 0; g < G; ++g) w[g] = n0 + g < N ? __ldg(W + (size_t)(n0 + g) * K + k) : 0.f;
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const float x = X[r * K + k];
#pragma unroll
                for (int g = 0; g < G; ++g) acc[g][r] = fmaf(x, w[g], acc[g][r]);
            }
        }
#pragma unroll
        for (int g = 0; g < G; ++g)
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const float v = smt_warp_sum(acc[g][r]);
                if (lane == 0 && n0 + g < N) {
                    const float o = v + __ldg(bias + n0 + g);
                    dst[r * N + n0 + g] = relu ? fmaxf(o, 0.f) : o;
                }
            }
    }
    __syncthreads();
}

// Y[r] = LN(Y[r] + R[r]) (R may be NULL), then optionally a second LN, for rows r < rows of shared-memory Y; one warp
// per row.  torch's LayerNorm: biased variance (two passes), (v - mean) / sqrt(var + eps) gamma + beta.  For the
// backward, U (row stride ldu) keeps the first LN's input and S (row stride lds) each pass's (mean, rstd); NULL skips.
__device__ void smt_row_norm(float* Y, int ldy, const float* R, size_t ldr, int rows, int d, SmtLn n1, SmtLn n2,
                             bool two, float* U = nullptr, size_t ldu = 0, float* S = nullptr, size_t lds = 0) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int r = warp; r < rows; r += SMT_THREADS / 32) {
        float* y = Y + (size_t)r * ldy;
        if (R)
            for (int c = lane; c < d; c += 32) y[c] += R[(size_t)r * ldr + c];
        __syncwarp();
        if (U)
            for (int c = lane; c < d; c += 32) U[(size_t)r * ldu + c] = y[c];
        for (int pass = 0; pass < (two ? 2 : 1); ++pass) {
            const float *g = pass ? n2.g : n1.g, *be = pass ? n2.b : n1.b, eps = pass ? n2.eps : n1.eps;
            float s = 0.f;
            for (int c = lane; c < d; c += 32) s += y[c];
            const float mean = smt_warp_sum(s) / (float)d;
            float q = 0.f;
            for (int c = lane; c < d; c += 32) {
                const float v = y[c] - mean;
                q = fmaf(v, v, q);
            }
            const float rstd = 1.f / sqrtf(smt_warp_sum(q) / (float)d + eps);
            if (S && lane == 0) {
                S[(size_t)r * lds + 2 * pass] = mean;
                S[(size_t)r * lds + 2 * pass + 1] = rstd;
            }
            __syncwarp();
            for (int c = lane; c < d; c += 32) y[c] = (y[c] - mean) * rstd * __ldg(g + c) + __ldg(be + c);
            __syncwarp();
        }
    }
    __syncthreads();
}

// sin and cos after a two-step reduction by 2 pi, on the hardware approximation (absolute error < 4e-7 on [-pi, pi]);
// the library's sinf / cosf would carry a local-memory slow path for huge arguments into the kernel.
__device__ __forceinline__ void smt_sincos(float x, float* s, float* c) {
    const float k = rintf(x * 0.159154943f);
    float r = fmaf(-k, 6.28318548f, x);                 // 2 pi rounded to float ...
    r = fmaf(-k, -1.74845553e-7f, r);                   // ... and what that rounding left out
    __sincosf(r, s, c);
}

// The 5 pose features [x, y, cos h, sin h, exp(-t)] of token pose q (x, y, heading, time) relative to the agent's p.
__device__ __forceinline__ void smt_pose_features(const float* p, const float* q, float* f) {
    const float ha = -p[2], hb = -q[2];
    const float dx = p[0] - q[0], dy = p[1] - q[1];
    const float rr = sqrtf(dx * dx + dy * dy);
    const float phi = atan2f(q[1] - p[1], q[0] - p[0]) - ha;
    float sp, cp, sd, cd, sh, ch;
    smt_sincos(phi, &sp, &cp);
    smt_sincos(hb - ha, &sd, &cd);
    smt_sincos(-atan2f(sd, cd), &sh, &ch);
    f[0] = rr * cp, f[1] = rr * sp, f[2] = ch, f[3] = sh, f[4] = expf(-q[3]);
}

// grid (ceil(T / SMT_RT), B).  Scans env b's mask (slot j is valid iff !((1 - mask) > 0), none under pretraining; the
// current token always), builds the CTA's 16 compacted rows [feat[:pi], pose_encoder(relative pose)] (or the raw rows
// without pose encoding) and writes fusion_encoder(rows) to h0.  CTA 0 of each env writes cnt[b].
__global__ void __launch_bounds__(SMT_THREADS, 1) smt_fuse_kernel(const SmtArgs a) {
    extern __shared__ __align__(16) float smt_smem[];
    float* smem = smt_smem;
    const int b = blockIdx.y, j0 = blockIdx.x * SMT_RT, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int Fp = (a.F + 3) & ~3;
    float* X = smem;                         // [RT][Fp]
    float* H1 = X + SMT_RT * Fp;             // [RT][d]
    float* Ws = H1 + SMT_RT * a.d;           // [SMT_WS]
    int* slot = (int*)(Ws + SMT_WS);         // [RT]
    int* wsum = slot + SMT_RT;               // [8]
    // four consecutive slots per thread (T <= 1024), exclusive scan over the block
    int v[4], c = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int j = tid * 4 + i;
        v[i] = j == a.M ? 1 : (j < a.M && !a.pretraining && !((1.f - a.masks[(size_t)b * a.M + j]) > 0.f));
        c += v[i];
    }
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) wsum[warp] = incl;
    if (tid < SMT_RT) slot[tid] = -1;
    __syncthreads();
    int pos = incl - c, total = 0;
    for (int w = 0; w < SMT_THREADS / 32; ++w) {
        if (w < warp) pos += wsum[w];
        total += wsum[w];
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
        if (v[i]) {
            if (pos >= j0 && pos < j0 + SMT_RT) slot[pos - j0] = tid * 4 + i;
            ++pos;
        }
    if (blockIdx.x == 0 && tid == 0) a.cnt[b] = total;
    __syncthreads();
    if (j0 >= total) return;
    const int rows = min(SMT_RT, total - j0);
    const size_t row0 = (size_t)b * a.T + j0;
    if (a.slot && tid < rows) a.slot[row0 + tid] = slot[tid];
    // input rows
    const int raw = a.pi >= 0 ? a.pi : a.d_in;
    for (int i = tid; i < SMT_RT * Fp; i += SMT_THREADS) {
        const int r = i / Fp, k = i % Fp;
        float val = 0.f;
        if (r < rows && k < raw) {
            const int s = slot[r];
            const float* src = s == a.M ? a.x + (size_t)b * a.d_in : a.memory + ((size_t)s * a.B + b) * a.d_in;
            val = src[k];
        }
        X[i] = val;
    }
    __syncthreads();
    if (a.pi >= 0 && tid < SMT_RT * 16) {
        const int r = tid / 16, o = tid % 16;
        if (r < rows) {
            const int s = slot[r];
            const float* p = a.x + (size_t)b * a.d_in + a.pi;
            const float* q = s == a.M ? p : a.memory + ((size_t)s * a.B + b) * a.d_in + a.pi;
            float f[5];
            smt_pose_features(p, q, f);
            const float* w = a.pose.w + o * 5;
            float e = 0.f;
#pragma unroll
            for (int i = 0; i < 5; ++i) e = fmaf(__ldg(w + i), f[i], e);
            X[r * Fp + a.pi + o] = e + __ldg(a.pose.b + o);
        }
    }
    __syncthreads();
    if (a.xin)
        for (int i = tid; i < rows * Fp; i += SMT_THREADS) a.xin[row0 * Fp + i] = X[i];
    smt_block_linear<SMT_RT, 2>(X, Fp, a.F, a.fuse1.w, a.fuse1.b, a.d, Ws, H1, a.d, SMT_RT, true);
    __syncthreads();
    if (a.hid)
        for (int i = tid; i < rows * a.d; i += SMT_THREADS) a.hid[row0 * a.d + i] = H1[i];
    smt_block_linear<SMT_RT, 2>(H1, a.d, a.d, a.fuse2.w, a.fuse2.b, a.d, Ws,
                                a.h0 + ((size_t)b * a.T + j0) * a.d, a.d, rows, false);
}

// grid (ceil(T / SMT_RT), ceil(N / 128), B): out rows [b][j][ldo] (columns n0 .. n0 + 127) = in rows W^T + bias for
// the env's valid rows j < cnt[b].
__global__ void __launch_bounds__(SMT_THREADS) smt_linear_kernel(const int* __restrict__ cnt, const float* in, int ldi,
                                                                 int T, int K, SmtLin lin, int N, float* out, int ldo) {
    extern __shared__ __align__(16) float smt_smem[];
    float* smem = smt_smem;
    const int b = blockIdx.z, j0 = blockIdx.x * SMT_RT, n0 = blockIdx.y * 128;
    const int rows = min(SMT_RT, cnt[b] - j0);
    if (rows <= 0) return;
    float* X = smem;                    // [RT][K]
    float* Ws = X + SMT_RT * K;
    const float* src = in + ((size_t)b * T + j0) * ldi;
    for (int i = threadIdx.x; i < SMT_RT * K; i += SMT_THREADS) {
        const int r = i / K, k = i % K;
        X[i] = r < rows ? src[(size_t)r * ldi + k] : 0.f;
    }
    __syncthreads();
    smt_block_linear<SMT_RT, 2>(X, K, K, lin.w + (size_t)n0 * K, lin.b + n0, min(128, N - n0), Ws,
                                out + ((size_t)b * T + j0) * ldo + n0, ldo, rows, false);
}

// Softmax attention of one query (shared-memory scores S[0..n)) over the env's n keys: p = exp(s - max) / sum, then
// out[c] = sum_j p_j V[j][c] in slot order; lane-owned output columns c = lane + 32 i < hd.
__device__ __forceinline__ void smt_softmax_pv(float* S, int n, const float* V, size_t ldv, int hd, float* out) {
    const int lane = threadIdx.x & 31;
    float m = -INFINITY;
    for (int j = lane; j < n; j += 32) m = fmaxf(m, S[j]);
    m = smt_warp_max(m);
    float s = 0.f;
    for (int j = lane; j < n; j += 32) {
        const float e = expf(S[j] - m);
        S[j] = e;
        s += e;
    }
    const float inv = 1.f / smt_warp_sum(s);
    __syncwarp();
    for (int c = lane; c < hd; c += 32) {
        float acc = 0.f;
        for (int j = 0; j < n; ++j) acc = fmaf(S[j] * inv, __ldg(V + (size_t)j * ldv + c), acc);
        out[c] = acc;
    }
    __syncwarp();
}

// grid (ceil(T / SMT_RT), H, B): queries j0 .. j0 + 15 of env b, head h, over the env's cnt[b] keys.  Scores go to
// S[16][T] (K staged through shared memory 64 keys at a time, one key per lane), then softmax and P.V per warp.
__global__ void __launch_bounds__(SMT_THREADS) smt_attn_kernel(const SmtArgs a) {
    extern __shared__ __align__(16) float smt_smem[];
    float* smem = smt_smem;
    const int b = blockIdx.z, h = blockIdx.y, j0 = blockIdx.x * SMT_RT, n = a.cnt[b];
    if (j0 >= n) return;
    const int hd = a.hd, ld3 = 3 * a.d, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int Tp = (a.T + 3) & ~3;
    float* Qs = smem;                         // [RT][hd]
    float* Ks = Qs + SMT_RT * hd;             // [64][hd + 1]
    float* S = Ks + SMT_KT_KEYS * (hd + 1);   // [RT][Tp]
    const float* base = a.qkv + (size_t)b * a.T * ld3;
    const float scale = 1.f / sqrtf((float)hd);
    for (int i = threadIdx.x; i < SMT_RT * hd; i += SMT_THREADS) {
        const int r = i / hd, c = i % hd;
        Qs[i] = j0 + r < n ? base[(size_t)(j0 + r) * ld3 + h * hd + c] : 0.f;
    }
    for (int k0 = 0; k0 < n; k0 += SMT_KT_KEYS) {
        const int kn = min(SMT_KT_KEYS, n - k0);
        __syncthreads();
        for (int i = threadIdx.x; i < kn * hd; i += SMT_THREADS) {
            const int r = i / hd, c = i % hd;
            Ks[r * (hd + 1) + c] = base[(size_t)(k0 + r) * ld3 + a.d + h * hd + c];
        }
        __syncthreads();
        for (int qi = warp; qi < SMT_RT; qi += SMT_THREADS / 32)
            for (int kj = lane; kj < kn; kj += 32) {
                const float* q = Qs + qi * hd;
                const float* k = Ks + kj * (hd + 1);
                float s = 0.f;
                for (int c = 0; c < hd; ++c) s = fmaf(q[c], k[c], s);
                S[qi * Tp + k0 + kj] = s * scale;
            }
    }
    __syncthreads();
    for (int qi = warp; qi < SMT_RT && j0 + qi < n; qi += SMT_THREADS / 32)
        smt_softmax_pv(S + qi * Tp, n, base + 2 * a.d + h * hd, ld3, hd, a.att + ((size_t)b * a.T + j0 + qi) * a.d + h * hd);
}

// grid (ceil(T / SMT_RT), B): E = encoder.norm(norm2(a + FF(a))), a = norm1(h0 + out_proj(att)), written to enc.
__global__ void __launch_bounds__(SMT_THREADS) smt_enc_tail_kernel(const SmtArgs a) {
    extern __shared__ __align__(16) float smt_smem[];
    float* smem = smt_smem;
    const int b = blockIdx.y, j0 = blockIdx.x * SMT_RT, d = a.d;
    const int rows = min(SMT_RT, a.cnt[b] - j0);
    if (rows <= 0) return;
    float* A = smem;                  // [RT][d]
    float* Y = A + SMT_RT * d;
    float* Z = Y + SMT_RT * d;
    float* Ws = Z + SMT_RT * d;
    const size_t row0 = (size_t)b * a.T + j0;
    const float* att = a.att + row0 * d;
    const float* h0 = a.h0 + row0 * d;
    float* u = a.u ? a.u + row0 * 2 * d : nullptr;
    float* st = a.st ? a.st + row0 * 6 : nullptr;
    for (int i = threadIdx.x; i < SMT_RT * d; i += SMT_THREADS) A[i] = i / d < rows ? att[i] : 0.f;
    __syncthreads();
    smt_block_linear<SMT_RT, 2>(A, d, d, a.enc_out.w, a.enc_out.b, d, Ws, Y, d, SMT_RT, false);
    __syncthreads();
    smt_row_norm(Y, d, h0, d, rows, d, a.enc_n1, a.enc_n1, false, u, 2 * d, st, 6);
    smt_block_linear<SMT_RT, 2>(Y, d, d, a.enc_ff1.w, a.enc_ff1.b, d, Ws, A, d, SMT_RT, true);
    __syncthreads();
    if (a.ffh)
        for (int i = threadIdx.x; i < rows * d; i += SMT_THREADS) a.ffh[row0 * d + i] = A[i];
    smt_block_linear<SMT_RT, 2>(A, d, d, a.enc_ff2.w, a.enc_ff2.b, d, Ws, Z, d, SMT_RT, false);
    __syncthreads();
    smt_row_norm(Z, d, Y, d, rows, d, a.enc_n2, a.enc_n, true, u ? u + d : nullptr, 2 * d, st ? st + 2 : nullptr, 6);
    for (int i = threadIdx.x; i < rows * d; i += SMT_THREADS) a.enc[row0 * d + i] = Z[i];
}

// grid ceil(B / SMT_DEC_ENVS): the decoder for envs e0 .. e0 + 3 with one target token each (goal, or the fused
// current token h0[b][cnt - 1]).  Self-attention over one key is out_proj(W_v t + b_v); cross-attention reads the
// K / V rows the K/V projection wrote into kv ([b][j][2d]).
__global__ void __launch_bounds__(SMT_THREADS, 1) smt_decoder_kernel(const SmtArgs a) {
    extern __shared__ __align__(16) float smt_smem[];
    float* smem = smt_smem;
    constexpr int R = SMT_DEC_ENVS;
    const int e0 = blockIdx.x * R, rows = min(R, a.B - e0), d = a.d, hd = a.hd;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, Tp = (a.T + 3) & ~3;
    float* T0 = smem;                 // [R][d]
    float* T1 = T0 + R * d;
    float* Q = T1 + R * d;
    float* Cc = Q + R * d;
    float* S = Cc + R * d;            // [8 warps][Tp]
    for (int i = threadIdx.x; i < R * d; i += SMT_THREADS) {
        const int r = i / d, c = i % d, b = e0 + r;
        float v = 0.f;
        if (r < rows)
            v = a.goal ? a.goal[(size_t)b * d + c] : a.h0[((size_t)b * a.T + a.cnt[b] - 1) * d + c];
        T0[i] = v;
    }
    __syncthreads();
    smt_rows_gemv<R>(T0, d, a.dec_v.w, a.dec_v.b, d, Q, false);
    __syncthreads();
    smt_rows_gemv<R>(Q, d, a.dec_sa_out.w, a.dec_sa_out.b, d, T1, false);
    __syncthreads();
    smt_row_norm(T1, d, T0, d, R, d, a.dec_n1, a.dec_n1, false);
    smt_rows_gemv<R>(T1, d, a.dec_q.w, a.dec_q.b, d, Q, false);
    __syncthreads();
    const float scale = 1.f / sqrtf((float)hd);
    float* Sw = S + warp * Tp;
    for (int p = warp; p < rows * a.H; p += SMT_THREADS / 32) {
        const int r = p / a.H, h = p % a.H, b = e0 + r, n = a.cnt[b];
        const float* kv = a.kv + (size_t)b * a.T * 2 * d;
        const float* q = Q + r * d + h * hd;
        for (int j = lane; j < n; j += 32) {
            const float* k = kv + (size_t)j * 2 * d + h * hd;
            float s = 0.f;
            for (int c = 0; c < hd; ++c) s = fmaf(q[c], __ldg(k + c), s);
            Sw[j] = s * scale;
        }
        __syncwarp();
        smt_softmax_pv(Sw, n, kv + d + h * hd, 2 * d, hd, Cc + r * d + h * hd);
    }
    __syncthreads();
    smt_rows_gemv<R>(Cc, d, a.dec_ca_out.w, a.dec_ca_out.b, d, T0, false);
    __syncthreads();
    smt_row_norm(T0, d, T1, d, R, d, a.dec_n2, a.dec_n2, false);
    smt_rows_gemv<R>(T0, d, a.dec_ff1.w, a.dec_ff1.b, d, Q, true);
    __syncthreads();
    smt_rows_gemv<R>(Q, d, a.dec_ff2.w, a.dec_ff2.b, d, T1, false);
    __syncthreads();
    smt_row_norm(T1, d, T0, d, rows, d, a.dec_n3, a.dec_n, true);
    for (int i = threadIdx.x; i < rows * d; i += SMT_THREADS) a.out[(size_t)e0 * d + i] = T1[i];
}

// ---------------------------------------------------------------------------
// The backward of the six launches above (ssb_smt_state_encoder_train_backward_batch), on the values the training
// forward kept (SmtArgs' slot / xin / hid / u / ffh / st, and att, qkv, kv, enc no longer overwritten).  Ten launches
// whatever B, M and the masks; CTAs past cnt[b] exit as in the forward:
//   smt_transpose_kernel   W^T of every Linear a dX goes through, and a zero bias (the dX GEMMs reuse the forward's)
//   smt_dec_bwd_kernel     recomputes the decoder (the same code as smt_decoder_kernel) and runs its reverse
//   smt_linear_kernel      dE = dKV W_kv (the K/V projection's reverse)
//   smt_enc_tail_bwd_kernel the tail's reverse: two LayerNorms, FF, norm1, out_proj -> datt and the residual's dh0
//   smt_attn_bwd_kernel<0> dQ per (env, head, 16 queries), recomputing the softmax from the saved Q / K
//   smt_attn_bwd_kernel<1> dK, dV per (env, head, 16 keys) over the env's queries
//   smt_linear_kernel      dh0 += dQKV W_qkv
//   smt_fuse_bwd_kernel    the fusion MLP's reverse, dx, and the pose encoding's reverse per token
//   smt_dw_kernel          every weight / bias / LayerNorm gradient as a row-split partial sum (split s: envs
//                          s B / S .. (s + 1) B / S, tokens in order)
//   smt_reduce_kernel      partials summed in split order; the decoder self-attention's Q / K rows (exactly 0); the
//                          agent pose's columns of dx summed over the env's tokens in order
// No float atomics: every output element is written by one thread, and every sum has a fixed order.
// ---------------------------------------------------------------------------
#define SMT_DW_SPLITS 32     // row splits of a weight-gradient sum
#define SMT_DW_TILE 64       // smt_dw_kernel: output tile (rows of dW) x (columns of dW, the bias column included)
#define SMT_MAX_TRAIN_ENVS 65535
#define SMT_N_WT 13          // transposed weights
#define SMT_SMEM_DEC_BWD ((14 * SMT_DEC_ENVS * SMT_MAX_D + 16 * SMT_MAX_TOKENS) * 4)
#define SMT_SMEM_ATTN_BWD (16 * SMT_MAX_TOKENS * 4)
#define SMT_SMEM_TAIL_BWD SMT_SMEM_TAIL
#define SMT_SMEM_FUSE_BWD ((2 * SMT_RT * SMT_MAX_D + SMT_RT * (SMT_MAX_IN + 16) + SMT_WS) * 4)

// one weight-gradient sum: dW[n][k] = sum_r dy[r][n] x[r][k] (k < K), db[n] = sum_r dy[r][n]; or, with diag, a
// LayerNorm's dgamma[c] = sum_r dy[r][c] x[r][c] (x: x-hat), dbeta[c] = sum_r dy[r][c].  Rows: each env's valid
// tokens (x / dy rows at (b T + j) ld), or one row per env (per_env: rows at b ld).
struct SmtDwJob {
    const float* x;
    const float* dy;
    float* part;           // [S][N][K + 1], diag: [S][2][N]
    float* outw;           // dW [N][K] or dgamma; NULL: not asked for
    float* outb;           // db [N] or dbeta
    int ldx, ldy, K, N, per_env, diag;
};

enum { SJ_FUSE1, SJ_FUSE2, SJ_QKV, SJ_OUT, SJ_FF1, SJ_FF2, SJ_KV, SJ_POSE, SJ_DV, SJ_DSAO, SJ_DQ, SJ_DCAO, SJ_DFF1,
       SJ_DFF2, SJ_EN1, SJ_EN2, SJ_EN, SJ_DN1, SJ_DN2, SJ_DN3, SJ_DN, SMT_JOBS };
// the decoder's per-env rows: X and dY of its six Linears, x-hat and dY of its four LayerNorms, d(target)
enum { SD_T0, SD_DV, SD_V, SD_DU1, SD_N1, SD_DQ, SD_CC, SD_DU2, SD_N2, SD_DFFP, SD_FF, SD_DU3, SD_XH1, SD_DY1, SD_XH2,
       SD_DY2, SD_XH3, SD_DY3, SD_XHN, SD_DYN, SD_DTGT, SMT_DEC_BUFS };

struct SmtBwdArgs {
    SmtArgs f;             // the forward's arguments, on the training workspace
    const float* dout;     // [B][ld_dout]
    int ld_dout, S;
    float *dkv, *dE, *datt, *du1, *du2, *dfp, *a1, *xn, *dn2, *x2, *da1, *x1, *dqkv, *dh0b, *dh0, *dhp, *dpe, *pf,
        *posec, *ast;      // per token ([B][T][...]); ast: [B][T][H][3] (max, 1 / sum, dO . O) per query and head
    float* dec[SMT_DEC_BUFS];   // [B][d] each
    const float* wt[SMT_N_WT];  // transposed weights
    const float* zeros;    // [3 d_model]
    float *dx, *dgoal;     // NULL: not asked for
    float *zero_w, *zero_b;     // dec.self_attn in_proj's Q / K rows of the gradient, NULL: not asked for
    SmtDwJob jobs[SMT_JOBS];
};
enum { SW_FUSE1, SW_FUSE2, SW_QKV, SW_OUT, SW_FF1, SW_FF2, SW_KV, SW_DV, SW_DSAO, SW_DQ, SW_DCAO, SW_DFF1, SW_DFF2 };

struct SmtTJob { const float* src; float* dst; int N, K; };
struct SmtTArgs { SmtTJob job[SMT_N_WT]; float* zeros; int nz; };

// grid (ceil(max N / 32) * ceil(max K / 32), SMT_N_WT): dst[k][n] = src[n][k] through a 32 x 33 tile.
__global__ void __launch_bounds__(SMT_THREADS) smt_transpose_kernel(__grid_constant__ const SmtTArgs t) {
    __shared__ float tile[32][33];
    if (blockIdx.x == 0 && blockIdx.y == 0)
        for (int i = threadIdx.x; i < t.nz; i += SMT_THREADS) t.zeros[i] = 0.f;
    const SmtTJob j = t.job[blockIdx.y];
    const int tk = (j.K + 31) / 32, n0 = blockIdx.x / tk * 32, k0 = blockIdx.x % tk * 32;
    if (n0 >= j.N) return;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int r = ty; r < 32; r += SMT_THREADS / 32)
        tile[r][tx] = n0 + r < j.N && k0 + tx < j.K ? j.src[(size_t)(n0 + r) * j.K + k0 + tx] : 0.f;
    __syncthreads();
    for (int r = ty; r < 32; r += SMT_THREADS / 32)
        if (k0 + r < j.K && n0 + tx < j.N) j.dst[(size_t)(k0 + r) * j.N + n0 + tx] = tile[tx][r];
}

// The reverse of smt_row_norm for rows r < rows of shared-memory G (in place: dY in, dU out), U and S as smt_row_norm
// kept them.  With two, the second LN's input is recomputed from U and the first pass's statistics.  x-hat and dY of
// each pass go to xh / dy (row stride ldo; NULL skips) for the gamma / beta sums.
__device__ void smt_row_norm_bwd(float* G, int ldg, const float* U, size_t ldu, const float* S, size_t lds, int rows,
                                 int d, SmtLn n1, SmtLn n2, bool two, float* xh1, float* dy1, float* xh2, float* dy2,
                                 size_t ldo) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int r = warp; r < rows; r += SMT_THREADS / 32) {
        float* g = G + (size_t)r * ldg;
        const float* u = U + (size_t)r * ldu;
        const float m1 = S[(size_t)r * lds], r1 = S[(size_t)r * lds + 1];
        for (int pass = two ? 1 : 0; pass >= 0; --pass) {
            const SmtLn n = pass ? n2 : n1;
            const float m2 = pass ? S[(size_t)r * lds + 2] : 0.f, r2 = pass ? S[(size_t)r * lds + 3] : 0.f;
            float* xo = pass ? xh2 : xh1;
            float* yo = pass ? dy2 : dy1;
            float sa = 0.f, sb = 0.f;
            for (int c = lane; c < d; c += 32) {
                float xh = (u[c] - m1) * r1;
                if (pass) xh = (xh * __ldg(n1.g + c) + __ldg(n1.b + c) - m2) * r2;
                const float gg = g[c] * __ldg(n.g + c);
                sa += gg;
                sb = fmaf(gg, xh, sb);
                if (xo) xo[(size_t)r * ldo + c] = xh;
                if (yo) yo[(size_t)r * ldo + c] = g[c];
            }
            sa = smt_warp_sum(sa) / (float)d;
            sb = smt_warp_sum(sb) / (float)d;
            const float rs = pass ? r2 : r1;
            __syncwarp();
            for (int c = lane; c < d; c += 32) {
                float xh = (u[c] - m1) * r1;
                if (pass) xh = (xh * __ldg(n1.g + c) + __ldg(n1.b + c) - m2) * r2;
                g[c] = rs * (g[c] * __ldg(n.g + c) - sa - xh * sb);
            }
            __syncwarp();
        }
    }
    __syncthreads();
}

// rows r < rows of shared-memory [R][d] src to global dst + r * d
__device__ __forceinline__ void smt_store_rows(const float* src, float* dst, int rows, int d) {
    for (int i = threadIdx.x; i < rows * d; i += SMT_THREADS) dst[i] = src[i];
}

// grid ceil(B / SMT_DEC_ENVS): the decoder of smt_decoder_kernel recomputed for envs e0 .. e0 + 3 (same code, same
// bits) keeping every intermediate, then its reverse from dout.  Writes dK / dV of the env's valid K/V rows (dkv),
// the per-env rows of the decoder's weight-gradient sums (dec[]) and d(target): dgoal, or dec[SD_DTGT] for the fused
// current token.  Self-attention over one key: softmax's gradient is exactly 0, so only W_v and out_proj get one.
__global__ void __launch_bounds__(SMT_THREADS, 1) smt_dec_bwd_kernel(__grid_constant__ const SmtBwdArgs g) {
    extern __shared__ __align__(16) float smt_smem[];
    const SmtArgs& a = g.f;
    constexpr int R = SMT_DEC_ENVS;
    const int e0 = blockIdx.x * R, rows = min(R, a.B - e0), d = a.d, hd = a.hd;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, Tp = (a.T + 3) & ~3;
    float* T0 = smt_smem;
    float* V = T0 + R * d;
    float* N1 = V + R * d;
    float* Q = N1 + R * d;
    float* Cc = Q + R * d;
    float* N2 = Cc + R * d;
    float* FF = N2 + R * d;
    float* N3 = FF + R * d;
    float* U = N3 + R * d;            // [3][R][d] LayerNorm inputs
    float* G = U + 3 * R * d;
    float* G2 = G + R * d;
    float* G3 = G2 + R * d;
    float* S = G3 + R * d;            // [8 warps][2][Tp]; 14 R d floats before it
    __shared__ float st[R][8];        // (mean, rstd) of norm1, norm2, norm3, decoder.norm
    for (int i = threadIdx.x; i < 14 * R * d; i += SMT_THREADS) smt_smem[i] = 0.f;
    __syncthreads();
    for (int i = threadIdx.x; i < R * d; i += SMT_THREADS) {
        const int r = i / d, c = i % d, b = e0 + r;
        float v = 0.f;
        if (r < rows)
            v = a.goal ? a.goal[(size_t)b * d + c] : a.h0[((size_t)b * a.T + a.cnt[b] - 1) * d + c];
        T0[i] = v;
        G[i] = r < rows ? g.dout[(size_t)b * g.ld_dout + c] : 0.f;
    }
    __syncthreads();
    smt_rows_gemv<R>(T0, d, a.dec_v.w, a.dec_v.b, d, V, false);
    __syncthreads();
    smt_rows_gemv<R>(V, d, a.dec_sa_out.w, a.dec_sa_out.b, d, N1, false);
    __syncthreads();
    smt_row_norm(N1, d, T0, d, R, d, a.dec_n1, a.dec_n1, false, U, d, &st[0][0], 8);
    smt_rows_gemv<R>(N1, d, a.dec_q.w, a.dec_q.b, d, Q, false);
    __syncthreads();
    const float scale = 1.f / sqrtf((float)hd);
    float* Sw = S + warp * 2 * Tp;
    float* Dw = Sw + Tp;
    for (int p = warp; p < rows * a.H; p += SMT_THREADS / 32) {
        const int r = p / a.H, h = p % a.H, b = e0 + r, n = a.cnt[b];
        const float* kv = a.kv + (size_t)b * a.T * 2 * d;
        const float* q = Q + r * d + h * hd;
        for (int j = lane; j < n; j += 32) {
            const float* k = kv + (size_t)j * 2 * d + h * hd;
            float s = 0.f;
            for (int c = 0; c < hd; ++c) s = fmaf(q[c], __ldg(k + c), s);
            Sw[j] = s * scale;
        }
        __syncwarp();
        smt_softmax_pv(Sw, n, kv + d + h * hd, 2 * d, hd, Cc + r * d + h * hd);
    }
    __syncthreads();
    smt_rows_gemv<R>(Cc, d, a.dec_ca_out.w, a.dec_ca_out.b, d, N2, false);
    __syncthreads();
    smt_row_norm(N2, d, N1, d, R, d, a.dec_n2, a.dec_n2, false, U + R * d, d, &st[0][2], 8);
    smt_rows_gemv<R>(N2, d, a.dec_ff1.w, a.dec_ff1.b, d, FF, true);
    __syncthreads();
    smt_rows_gemv<R>(FF, d, a.dec_ff2.w, a.dec_ff2.b, d, N3, false);
    __syncthreads();
    smt_row_norm(N3, d, N2, d, R, d, a.dec_n3, a.dec_n, true, U + 2 * R * d, d, &st[0][4], 8);
    // reverse
    float* const* D = g.dec;
    const size_t o = (size_t)e0 * d;
    smt_row_norm_bwd(G, d, U + 2 * R * d, d, &st[0][4], 8, rows, d, a.dec_n3, a.dec_n, true, D[SD_XH3] + o,
                     D[SD_DY3] + o, D[SD_XHN] + o, D[SD_DYN] + o, d);
    smt_rows_gemv<R>(G, d, g.wt[SW_DFF2], g.zeros, d, G2, false);
    for (int i = threadIdx.x; i < R * d; i += SMT_THREADS) G2[i] = FF[i] > 0.f ? G2[i] : 0.f;
    __syncthreads();
    smt_rows_gemv<R>(G2, d, g.wt[SW_DFF1], g.zeros, d, G3, false);
    smt_store_rows(G, D[SD_DU3] + o, rows, d);
    smt_store_rows(FF, D[SD_FF] + o, rows, d);
    smt_store_rows(G2, D[SD_DFFP] + o, rows, d);
    smt_store_rows(N2, D[SD_N2] + o, rows, d);
    for (int i = threadIdx.x; i < R * d; i += SMT_THREADS) G[i] += G3[i];
    __syncthreads();
    smt_row_norm_bwd(G, d, U + R * d, d, &st[0][2], 8, rows, d, a.dec_n2, a.dec_n2, false, D[SD_XH2] + o,
                     D[SD_DY2] + o, nullptr, nullptr, d);
    smt_rows_gemv<R>(G, d, g.wt[SW_DCAO], g.zeros, d, G2, false);     // dCc
    smt_store_rows(G, D[SD_DU2] + o, rows, d);
    smt_store_rows(Cc, D[SD_CC] + o, rows, d);
    // cross-attention: dQ to G3, dK / dV of the env's valid rows to dkv
    for (int p = warp; p < rows * a.H; p += SMT_THREADS / 32) {
        const int r = p / a.H, h = p % a.H, b = e0 + r, n = a.cnt[b];
        const float* kv = a.kv + (size_t)b * a.T * 2 * d;
        float* dkv = g.dkv + (size_t)b * a.T * 2 * d;
        const float* q = Q + r * d + h * hd;
        const float* dc = G2 + r * d + h * hd;
        float m = -INFINITY;
        for (int j = lane; j < n; j += 32) {
            const float* k = kv + (size_t)j * 2 * d + h * hd;
            float s = 0.f;
            for (int c = 0; c < hd; ++c) s = fmaf(q[c], __ldg(k + c), s);
            Sw[j] = s * scale;
            m = fmaxf(m, Sw[j]);
        }
        m = smt_warp_max(m);
        float sum = 0.f;
        for (int j = lane; j < n; j += 32) {
            const float e = expf(Sw[j] - m);
            Sw[j] = e;
            sum += e;
        }
        const float inv = 1.f / smt_warp_sum(sum);
        float dsum = 0.f;
        for (int j = lane; j < n; j += 32) {
            const float* v = kv + (size_t)j * 2 * d + d + h * hd;
            float dp = 0.f;
            for (int c = 0; c < hd; ++c) dp = fmaf(dc[c], __ldg(v + c), dp);
            Sw[j] *= inv;
            Dw[j] = dp;
            dsum = fmaf(Sw[j], dp, dsum);
        }
        dsum = smt_warp_sum(dsum);
        for (int j = lane; j < n; j += 32) Dw[j] = Sw[j] * (Dw[j] - dsum);
        __syncwarp();
        for (int c = lane; c < hd; c += 32) {
            float acc = 0.f;
            for (int j = 0; j < n; ++j) acc = fmaf(Dw[j], __ldg(kv + (size_t)j * 2 * d + h * hd + c), acc);
            G3[r * d + h * hd + c] = acc * scale;
            for (int j = 0; j < n; ++j) {
                dkv[(size_t)j * 2 * d + h * hd + c] = Dw[j] * scale * q[c];
                dkv[(size_t)j * 2 * d + d + h * hd + c] = Sw[j] * dc[c];
            }
        }
        __syncwarp();
    }
    __syncthreads();
    smt_rows_gemv<R>(G3, d, g.wt[SW_DQ], g.zeros, d, G2, false);
    smt_store_rows(G3, D[SD_DQ] + o, rows, d);
    smt_store_rows(N1, D[SD_N1] + o, rows, d);
    for (int i = threadIdx.x; i < R * d; i += SMT_THREADS) G[i] += G2[i];
    __syncthreads();
    smt_row_norm_bwd(G, d, U, d, &st[0][0], 8, rows, d, a.dec_n1, a.dec_n1, false, D[SD_XH1] + o, D[SD_DY1] + o,
                     nullptr, nullptr, d);
    smt_rows_gemv<R>(G, d, g.wt[SW_DSAO], g.zeros, d, G2, false);     // dV
    smt_rows_gemv<R>(G2, d, g.wt[SW_DV], g.zeros, d, G3, false);
    smt_store_rows(G, D[SD_DU1] + o, rows, d);
    smt_store_rows(V, D[SD_V] + o, rows, d);
    smt_store_rows(G2, D[SD_DV] + o, rows, d);
    smt_store_rows(T0, D[SD_T0] + o, rows, d);
    float* dt = a.goal ? g.dgoal : D[SD_DTGT];
    if (dt)
        for (int i = threadIdx.x; i < rows * d; i += SMT_THREADS) dt[o + i] = G[i] + G3[i];
}

// grid (ceil(T / SMT_RT), B): the reverse of smt_enc_tail_kernel for the env's valid rows j0 .. j0 + 15, from dE.
__global__ void __launch_bounds__(SMT_THREADS) smt_enc_tail_bwd_kernel(__grid_constant__ const SmtBwdArgs g) {
    extern __shared__ __align__(16) float smt_smem[];
    const SmtArgs& a = g.f;
    const int b = blockIdx.y, j0 = blockIdx.x * SMT_RT, d = a.d;
    const int rows = min(SMT_RT, a.cnt[b] - j0);
    if (rows <= 0) return;
    float* G = smt_smem;              // [RT][d]
    float* G2 = G + SMT_RT * d;
    float* G3 = G2 + SMT_RT * d;
    float* Ws = G3 + SMT_RT * d;
    const size_t row0 = (size_t)b * a.T + j0, o = row0 * d;
    const float* u = a.u + row0 * 2 * d;
    const float* st = a.st + row0 * 6;
    for (int i = threadIdx.x; i < SMT_RT * d; i += SMT_THREADS) G[i] = i / d < rows ? g.dE[o + i] : 0.f;
    __syncthreads();
    smt_row_norm_bwd(G, d, u + d, 2 * d, st + 2, 6, rows, d, a.enc_n2, a.enc_n, true, g.x2 + o, g.dn2 + o, g.xn + o,
                     nullptr, d);
    smt_store_rows(G, g.du2 + o, rows, d);
    smt_block_linear<SMT_RT, 2>(G, d, d, g.wt[SW_FF2], g.zeros, d, Ws, G2, d, SMT_RT, false);
    __syncthreads();
    for (int i = threadIdx.x; i < SMT_RT * d; i += SMT_THREADS) {
        const int r = i / d;
        G2[i] = r < rows && a.ffh[o + i] > 0.f ? G2[i] : 0.f;
        if (r < rows) {
            const int c = i % d;
            g.a1[o + i] = (u[(size_t)r * 2 * d + c] - st[r * 6]) * st[r * 6 + 1] * __ldg(a.enc_n1.g + c) +
                          __ldg(a.enc_n1.b + c);
        }
    }
    __syncthreads();
    smt_store_rows(G2, g.dfp + o, rows, d);
    smt_block_linear<SMT_RT, 2>(G2, d, d, g.wt[SW_FF1], g.zeros, d, Ws, G3, d, SMT_RT, false);
    __syncthreads();
    for (int i = threadIdx.x; i < SMT_RT * d; i += SMT_THREADS) G[i] += G3[i];
    __syncthreads();
    smt_row_norm_bwd(G, d, u, 2 * d, st, 6, rows, d, a.enc_n1, a.enc_n1, false, g.x1 + o, g.da1 + o, nullptr, nullptr,
                     d);
    smt_store_rows(G, g.du1 + o, rows, d);
    smt_block_linear<SMT_RT, 2>(G, d, d, g.wt[SW_OUT], g.zeros, d, Ws, g.datt + o, d, rows, false);
}

// grid (ceil(T / SMT_RT), H, B).  KV = false: queries j0 .. j0 + 15 of env b, head h: the scores and softmax as
// smt_attn_kernel computes them, dP = dO . V, D = sum_j P dP, dS = P (dP - D), dQ = scale sum_j dS K; keeps (max,
// 1 / sum, D) per query.  KV = true: keys j0 .. j0 + 15: dV = sum_i P dO, dK = scale sum_i dS Q over the env's
// queries in order.  One warp per query / key; rows of qkv, datt read through L1.
template <bool KV>
__global__ void __launch_bounds__(SMT_THREADS) smt_attn_bwd_kernel(__grid_constant__ const SmtBwdArgs g) {
    extern __shared__ __align__(16) float smt_smem[];
    const SmtArgs& a = g.f;
    const int b = blockIdx.z, h = blockIdx.y, j0 = blockIdx.x * SMT_RT, n = a.cnt[b];
    if (j0 >= n) return;
    const int hd = a.hd, d = a.d, ld3 = 3 * d, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, H = a.H;
    const int Tp = (a.T + 3) & ~3;
    float* Sw = smt_smem + warp * 2 * Tp;
    float* Dw = Sw + Tp;
    const float* base = a.qkv + (size_t)b * a.T * ld3;
    const float* dO = g.datt + (size_t)b * a.T * d + h * hd;
    float* ast = g.ast + (size_t)b * a.T * H * 3;
    float* dq = g.dqkv + (size_t)b * a.T * ld3;
    const float scale = 1.f / sqrtf((float)hd);
    for (int t = j0 + warp; t < min(j0 + SMT_RT, n); t += SMT_THREADS / 32) {
        if (!KV) {
            const float* q = base + (size_t)t * ld3 + h * hd;
            const float* go = dO + (size_t)t * d;
            float m = -INFINITY;
            for (int j = lane; j < n; j += 32) {
                const float* k = base + (size_t)j * ld3 + d + h * hd;
                float s = 0.f;
                for (int c = 0; c < hd; ++c) s = fmaf(q[c], k[c], s);
                Sw[j] = s * scale;
                m = fmaxf(m, Sw[j]);
            }
            m = smt_warp_max(m);
            float sum = 0.f;
            for (int j = lane; j < n; j += 32) {
                const float e = expf(Sw[j] - m);
                Sw[j] = e;
                sum += e;
            }
            const float inv = 1.f / smt_warp_sum(sum);
            float dsum = 0.f;
            for (int j = lane; j < n; j += 32) {
                const float* v = base + (size_t)j * ld3 + 2 * d + h * hd;
                float dp = 0.f;
                for (int c = 0; c < hd; ++c) dp = fmaf(go[c], v[c], dp);
                Sw[j] *= inv;
                Dw[j] = dp;
                dsum = fmaf(Sw[j], dp, dsum);
            }
            dsum = smt_warp_sum(dsum);
            for (int j = lane; j < n; j += 32) Dw[j] = Sw[j] * (Dw[j] - dsum);
            if (lane == 0) {
                float* s3 = ast + ((size_t)t * H + h) * 3;
                s3[0] = m, s3[1] = inv, s3[2] = dsum;
            }
            __syncwarp();
            for (int c = lane; c < hd; c += 32) {
                float acc = 0.f;
                for (int j = 0; j < n; ++j) acc = fmaf(Dw[j], base[(size_t)j * ld3 + d + h * hd + c], acc);
                dq[(size_t)t * ld3 + h * hd + c] = acc * scale;
            }
        } else {
            const float* k = base + (size_t)t * ld3 + d + h * hd;
            const float* v = base + (size_t)t * ld3 + 2 * d + h * hd;
            for (int i = lane; i < n; i += 32) {
                const float* q = base + (size_t)i * ld3 + h * hd;
                const float* go = dO + (size_t)i * d;
                const float* s3 = ast + ((size_t)i * H + h) * 3;
                float s = 0.f, dp = 0.f;
                for (int c = 0; c < hd; ++c) s = fmaf(q[c], k[c], s);
                for (int c = 0; c < hd; ++c) dp = fmaf(go[c], v[c], dp);
                const float p = expf(s * scale - s3[0]) * s3[1];
                Sw[i] = p;
                Dw[i] = p * (dp - s3[2]);
            }
            __syncwarp();
            for (int c = lane; c < hd; c += 32) {
                float dv = 0.f, dk = 0.f;
                for (int i = 0; i < n; ++i) {
                    dv = fmaf(Sw[i], dO[(size_t)i * d + c], dv);
                    dk = fmaf(Dw[i], base[(size_t)i * ld3 + h * hd + c], dk);
                }
                dq[(size_t)t * ld3 + d + h * hd + c] = dk * scale;
                dq[(size_t)t * ld3 + 2 * d + h * hd + c] = dv;
            }
        }
        __syncwarp();
    }
}

// The agent pose's gradient (x, y, heading, time) from token row pose q (the agent's own pose p when cur) through
// smt_pose_features, given the features' gradient gf.  As torch's autograd of the reference: 0 through r and atan2
// at r = 0, the heading terms of the current token cancel, and time reaches the agent from its own token only.
__device__ void smt_pose_features_bwd(const float* p, const float* q, bool cur, const float* gf, float* gp) {
    const float ha = -p[2], hb = -q[2];
    const float dx = p[0] - q[0], dy = p[1] - q[1];
    const float rr = sqrtf(dx * dx + dy * dy);
    const float phi = atan2f(q[1] - p[1], q[0] - p[0]) - ha;
    float sp, cp, sd, cd, sh, ch;
    smt_sincos(phi, &sp, &cp);
    smt_sincos(hb - ha, &sd, &cd);
    smt_sincos(-atan2f(sd, cd), &sh, &ch);
    gp[0] = gp[1] = gp[2] = gp[3] = 0.f;
    if (cur) {
        gp[3] = -gf[4] * expf(-q[3]);
        return;
    }
    gp[2] = -(-gf[2] * sh + gf[3] * ch);                  // heading: d(-atan2(sin, cos)) / d(hb - ha) = -1
    if (rr > 0.f) {
        const float gr = gf[0] * cp + gf[1] * sp, gphi = rr * (gf[1] * cp - gf[0] * sp);
        const float ex = q[0] - p[0], ey = q[1] - p[1], den = ex * ex + ey * ey;
        gp[0] = gr * dx / rr + gphi * ey / den;
        gp[1] = gr * dy / rr - gphi * ex / den;
        gp[2] += gphi;
    }
}

// grid (ceil(T / SMT_RT), B): the reverse of smt_fuse_kernel for the env's valid rows.  dh0 = the tail's residual
// gradient + the QKV rows' + (without a goal) d(target) on the current token; then fusion_encoder's two Linears;
// dx's feature columns from the current token's row; per token the pose_encoder's rows (dpe, features pf) and the
// agent pose's share (posec), which smt_reduce_kernel sums.
__global__ void __launch_bounds__(SMT_THREADS) smt_fuse_bwd_kernel(__grid_constant__ const SmtBwdArgs g) {
    extern __shared__ __align__(16) float smt_smem[];
    const SmtArgs& a = g.f;
    const int b = blockIdx.y, j0 = blockIdx.x * SMT_RT, d = a.d, n = a.cnt[b];
    const int rows = min(SMT_RT, n - j0);
    if (rows <= 0) return;
    const int Fp = (a.F + 3) & ~3;
    float* G = smt_smem;              // [RT][d]
    float* G2 = G + SMT_RT * d;       // [RT][d]
    float* DX = G2 + SMT_RT * d;      // [RT][Fp]
    float* Ws = DX + SMT_RT * Fp;
    const size_t row0 = (size_t)b * a.T + j0, o = row0 * d;
    const float* dt = g.dec[SD_DTGT] + (size_t)b * d;
    for (int i = threadIdx.x; i < SMT_RT * d; i += SMT_THREADS) {
        const int r = i / d;
        float v = 0.f;
        if (r < rows) {
            v = g.du1[o + i] + g.dh0b[o + i];
            if (!a.goal && j0 + r == n - 1) v += dt[i % d];
        }
        G[i] = v;
    }
    __syncthreads();
    smt_store_rows(G, g.dh0 + o, rows, d);
    smt_block_linear<SMT_RT, 2>(G, d, d, g.wt[SW_FUSE2], g.zeros, d, Ws, G2, d, SMT_RT, false);
    __syncthreads();
    for (int i = threadIdx.x; i < SMT_RT * d; i += SMT_THREADS)
        G2[i] = i / d < rows && a.hid[o + i] > 0.f ? G2[i] : 0.f;
    __syncthreads();
    smt_store_rows(G2, g.dhp + o, rows, d);
    smt_block_linear<SMT_RT, 2>(G2, d, d, g.wt[SW_FUSE1], g.zeros, a.F, Ws, DX, Fp, SMT_RT, false);
    __syncthreads();
    const int cur = n - 1 - j0;
    const int raw = a.pi >= 0 ? a.pi : a.d_in;
    if (g.dx && cur < rows)
        for (int k = threadIdx.x; k < raw; k += SMT_THREADS) g.dx[(size_t)b * a.d_in + k] = DX[cur * Fp + k];
    if (a.pi >= 0 && threadIdx.x < rows) {
        const int r = threadIdx.x, s = a.slot[row0 + r];
        const float* p = a.x + (size_t)b * a.d_in + a.pi;
        const float* q = s == a.M ? p : a.memory + ((size_t)s * a.B + b) * a.d_in + a.pi;
        float f[5], gf[5] = {0.f, 0.f, 0.f, 0.f, 0.f}, gp[4];
        smt_pose_features(p, q, f);
        for (int k = 0; k < 16; ++k) {
            const float e = DX[r * Fp + a.pi + k];
            g.dpe[(row0 + r) * 16 + k] = e;
            for (int i = 0; i < 5; ++i) gf[i] = fmaf(e, __ldg(a.pose.w + k * 5 + i), gf[i]);
        }
        for (int i = 0; i < 5; ++i) g.pf[(row0 + r) * 8 + i] = f[i];
        smt_pose_features_bwd(p, q, s == a.M, gf, gp);
        for (int i = 0; i < 4; ++i) g.posec[(row0 + r) * 4 + i] = gp[i];
    }
}

// grid (max tiles, S, SMT_JOBS): split s of job z (see SmtDwJob), tile blockIdx.x of its [N][K + 1] output (the
// bias as a column of ones), or 256 columns of a LayerNorm's (dgamma, dbeta).  Rows in env order, tokens in order.
__global__ void __launch_bounds__(SMT_THREADS) smt_dw_kernel(__grid_constant__ const SmtBwdArgs g) {
    __shared__ float Ys[16][SMT_DW_TILE + 1], Xs[16][SMT_DW_TILE + 1];
    const SmtDwJob& jb = g.jobs[blockIdx.z];
    if (!jb.part || jb.N == 0) return;
    const SmtArgs& a = g.f;
    const int s = blockIdx.y, b0 = (int)((long long)s * a.B / g.S), b1 = (int)((long long)(s + 1) * a.B / g.S);
    const int tid = threadIdx.x;
    auto row = [&](const float* p, int ld, int b, int j) {
        return p + (jb.per_env ? (size_t)b : (size_t)b * a.T + j) * ld;
    };
    if (jb.diag) {
        const int c = blockIdx.x * SMT_THREADS + tid;
        if (blockIdx.x * SMT_THREADS >= jb.N) return;
        float sg = 0.f, sb = 0.f;
        if (c < jb.N)
            for (int b = b0; b < b1; ++b) {
                const int nb = jb.per_env ? 1 : a.cnt[b];
                for (int t0 = 0; t0 < nb; t0 += 16) {       // 16-row partial sums, then their sum
                    float cg = 0.f, cb = 0.f;
                    for (int j = t0; j < min(nb, t0 + 16); ++j) {
                        const float y = row(jb.dy, jb.ldy, b, j)[c];
                        cg = fmaf(y, row(jb.x, jb.ldx, b, j)[c], cg);
                        cb += y;
                    }
                    sg += cg, sb += cb;
                }
            }
        if (c < jb.N) {
            jb.part[((size_t)s * 2) * jb.N + c] = sg;
            jb.part[((size_t)s * 2 + 1) * jb.N + c] = sb;
        }
        return;
    }
    const int K1 = jb.K + 1, tk = (K1 + SMT_DW_TILE - 1) / SMT_DW_TILE;
    const int n0 = blockIdx.x / tk * SMT_DW_TILE, k0 = blockIdx.x % tk * SMT_DW_TILE;
    if (n0 >= jb.N) return;
    const int ty = tid / 16, tx = tid % 16;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int b = b0; b < b1; ++b) {
        const int nb = jb.per_env ? 1 : a.cnt[b];
        for (int t0 = 0; t0 < nb; t0 += 16) {
            for (int i = tid; i < 16 * SMT_DW_TILE; i += SMT_THREADS) {
                const int r = i / SMT_DW_TILE, c = i % SMT_DW_TILE;
                const bool ok = t0 + r < nb;
                Ys[r][c] = ok && n0 + c < jb.N ? row(jb.dy, jb.ldy, b, t0 + r)[n0 + c] : 0.f;
                Xs[r][c] = !ok ? 0.f : k0 + c < jb.K ? row(jb.x, jb.ldx, b, t0 + r)[k0 + c] : k0 + c == jb.K ? 1.f : 0.f;
            }
            __syncthreads();
            float c[4][4];                                  // the 16 rows' partial sum, then added to acc
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) c[i][j] = 0.f;
#pragma unroll 4
            for (int r = 0; r < 16; ++r) {
                float y[4], x[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) y[i] = Ys[r][ty + 16 * i], x[i] = Xs[r][tx + 16 * i];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) c[i][j] = fmaf(y[i], x[j], c[i][j]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] += c[i][j];
            __syncthreads();
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int nn = n0 + ty + 16 * i, kk = k0 + tx + 16 * j;
            if (nn < jb.N && kk < K1) jb.part[((size_t)s * jb.N + nn) * K1 + kk] = acc[i][j];
        }
}

// grid (ceil(max elements / 256), SMT_JOBS + 2): job z's partials summed over the S splits in order into its
// outputs; z = SMT_JOBS: zeros into dec.self_attn's in_proj Q / K rows; z = SMT_JOBS + 1: dx's pose columns, the
// per-token shares summed over the env's tokens in order (0 past the 4 pose columns).
__global__ void __launch_bounds__(SMT_THREADS) smt_reduce_kernel(__grid_constant__ const SmtBwdArgs g) {
    const SmtArgs& a = g.f;
    const size_t e = (size_t)blockIdx.x * SMT_THREADS + threadIdx.x;
    if (blockIdx.y == SMT_JOBS) {
        const size_t nw = 2 * (size_t)a.d * a.d;
        if (g.zero_w && e < nw) g.zero_w[e] = 0.f;
        if (g.zero_b && e < 2 * (size_t)a.d) g.zero_b[e] = 0.f;
        return;
    }
    if (blockIdx.y == SMT_JOBS + 1) {
        if (a.pi < 0 || !g.dx) return;
        const int w = a.d_in - a.pi;
        if (e >= (size_t)a.B * w) return;
        const int b = (int)(e / w), c = (int)(e % w);
        float v = 0.f;
        if (c < 4)
            for (int j = 0; j < a.cnt[b]; ++j) v += g.posec[((size_t)b * a.T + j) * 4 + c];
        g.dx[(size_t)b * a.d_in + a.pi + c] = v;
        return;
    }
    const SmtDwJob& jb = g.jobs[blockIdx.y];
    if (!jb.part || jb.N == 0) return;
    const size_t per = jb.diag ? 2 * (size_t)jb.N : (size_t)jb.N * (jb.K + 1);
    if (e >= per) return;
    float v = 0.f;
    for (int s = 0; s < g.S; ++s) v += jb.part[s * per + e];
    if (jb.diag) {
        float* out = e < (size_t)jb.N ? jb.outw : jb.outb;
        if (out) out[e % jb.N] = v;
    } else {
        const int n = (int)(e / (jb.K + 1)), k = (int)(e % (jb.K + 1));
        if (k < jb.K) {
            if (jb.outw) jb.outw[(size_t)n * jb.K + k] = v;
        } else if (jb.outb) {
            jb.outb[n] = v;
        }
    }
}

__global__ void pcm16_decode_kernel(const int16_t* __restrict__ in, long long n, float* __restrict__ out) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long step = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += step) out[i] = (float)in[i] * (1.0f / 32768.0f);
}

__global__ void pcm16_encode_kernel(const float* __restrict__ in, long long n, int mode, int16_t* __restrict__ out) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long step = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += step) {
        float x = in[i];
        float v = mode == 0 ? rintf(x * 32768.0f) : truncf(x * 32767.0f);
        v = fminf(fmaxf(v, -32768.0f), 32767.0f);
        out[i] = (int16_t)(int)v;
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
// mac_ifft_cluster_kernel (N = 4096): the receive buffers a CTA holds at once.  Three of 34 KB keep two 256-thread CTAs
// (128 registers each) per SM and take config 2's 22 blocks in one round with 8-CTA clusters.
constexpr int kMacRoundBlocks = 3;

// CTAs per env of mac_ifft_cluster_kernel: the largest power of two <= min(8, n_blocks), so every rank owns a block
static int mac_cluster_size(int n_blocks) {
    int cl = 1;
    while (cl < 8 && 2 * cl <= n_blocks) cl *= 2;
    return cl;
}

template <int CL>
static cudaError_t set_cluster_smem_attr() {
    return cudaFuncSetAttribute(mac_ifft_cluster_kernel<12, CL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                kMacRoundBlocks * FftPlan<12>::SMEM_ELEMS * (int)sizeof(float2));
}

template <int LOG2N>
static int setup_smem_attrs() {
    using P = FftPlan<LOG2N>;
    const int bytes = (P::SMEM_ELEMS + P::TW_SMALL_ELEMS) * (int)sizeof(float2);
    cudaError_t e = cudaFuncSetAttribute(fwd_rir_kernel<LOG2N>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(fwd_src_kernel<LOG2N>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(mac_ifft_kernel<LOG2N, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if constexpr (LOG2N == 12) {          // conv_mode 0 schedules, as launch_conv_sub picks them
        if (e == cudaSuccess) e = set_cluster_smem_attr<1>();
        if (e == cudaSuccess) e = set_cluster_smem_attr<2>();
        if (e == cudaSuccess) e = set_cluster_smem_attr<4>();
        if (e == cudaSuccess) e = set_cluster_smem_attr<8>();
    } else {
        if (e == cudaSuccess) e = cudaFuncSetAttribute(mac_ifft_kernel<LOG2N, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    }
    return e == cudaSuccess ? 0 : -1;
}

// twiddle table of FftPlan<LOG2N>: pass p, rows e in {1,2,3,4,8,12}: [row][j] = exp(-2 pi i j e / (16 stride(p))),
// computed in double and rounded once
template <int LOG2N>
static cudaError_t upload_twiddles(ssb_ctx* ctx) {
    using P = FftPlan<LOG2N>;
    static const int kExp[6] = {1, 2, 3, 4, 8, 12};
    std::vector<float2> h(P::TW_ELEMS);
    for (int p = 0; p < P::NPASS; ++p) {
        const int st = P::stride(p);
        for (int row = 0; row < 6; ++row)
            for (int j = 0; j < st; ++j) {
                const double a = -2.0 * M_PI * (double)j * (double)kExp[row] / (16.0 * (double)st);
                h[P::tw_offset(p) + row * st + j] = make_float2((float)cos(a), (float)sin(a));
            }
    }
    cudaError_t e = cudaMalloc(&ctx->tw[LOG2N], h.size() * sizeof(float2));
    if (e == cudaSuccess) e = cudaMemcpy(ctx->tw[LOG2N], h.data(), h.size() * sizeof(float2), cudaMemcpyHostToDevice);
    return e;
}

// Grows a context-owned device scratch buffer to at least `need` float2; it never shrinks.  Kernels queued on any
// stream may still read the old buffer, so the device is synchronised before it is freed.
static cudaError_t grow_scratch(float2*& buf, size_t& elems, size_t need) {
    if (need <= elems) return cudaSuccess;
    if (buf) {
        cudaDeviceSynchronize();
        cudaFree(buf);
        buf = nullptr;
        elems = 0;
    }
    cudaError_t e = cudaMalloc(&buf, need * sizeof(float2));
    if (e == cudaSuccess) elems = need;
    return e;
}

extern "C" int ssb_version(void) { return 100; }

extern "C" int ssb_create(int device, ssb_ctx** out) {
    if (!out) return SSB_E_INVALID_ARG;
    *out = nullptr;
    ssb_ctx* ctx = new (std::nothrow) ssb_ctx();
    if (!ctx) return SSB_E_OOM;
    memset(ctx, 0, sizeof(*ctx));
    ctx->device = device;
    ctx->timed = new (std::nothrow) std::vector<TimedLaunch>();
    ctx->mel = new (std::nothrow) std::vector<ssb_ctx::MelBank>();
    *out = ctx;   // returned even on failure so that ssb_last_error works; caller destroys
    if (!ctx->timed || !ctx->mel) SSB_FAIL(ctx, SSB_E_OOM, "out of host memory");
    return abi_call(ctx, [&]() -> int {   // the caller's current device is restored
        {   // abi_call's guard has already selected the device; surface a bad ordinal as an error
            int cur = -1;
            SSB_CUDA(ctx, cudaGetDevice(&cur));
            if (cur != device) SSB_CUDA(ctx, cudaSetDevice(device));
        }
        cudaDeviceProp prop;
        SSB_CUDA(ctx, cudaGetDeviceProperties(&prop, device));
        if (prop.major != 9 || prop.minor != 0)
            SSB_FAIL(ctx, SSB_E_CUDA, "device %d is sm_%d%d; libssb200 is built for sm_90a only", device, prop.major, prop.minor);
        ctx->sm_count = prop.multiProcessorCount;
        ctx->n_streams = 2;
        ctx->n_chunks = 1;
        {
            cudaError_t e = cudaSuccess;
            if (e == cudaSuccess) e = upload_twiddles<9>(ctx);
            if (e == cudaSuccess) e = upload_twiddles<12>(ctx);
            if (e == cudaSuccess) e = upload_twiddles<13>(ctx);
            if (e == cudaSuccess) e = upload_twiddles<14>(ctx);
            SSB_CUDA(ctx, e);
        }
        {
            float hw[SSB_N_FFT];
            const int lpad = (SSB_N_FFT - SSB_WIN) / 2;
            for (int i = 0; i < SSB_N_FFT; ++i) hw[i] = 0.f;
            // scipy.signal.get_window('hann', 400, fftbins=True): 0.5 - 0.5 cos(2 pi n / 400)
            for (int n = 0; n < SSB_WIN; ++n) hw[lpad + n] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * (double)n / (double)SSB_WIN));
            SSB_CUDA(ctx, cudaMalloc(&ctx->window, sizeof(hw)));
            SSB_CUDA(ctx, cudaMemcpy(ctx->window, hw, sizeof(hw), cudaMemcpyHostToDevice));
        }
        {   // single-block plan: w_64 constants (per-device constant memory), the [16][1024] modulation table, smem opt-in
            float2 w64[64];
            for (int k = 0; k < 64; ++k) {
                const double a = -2.0 * M_PI * (double)k / 64.0;
                w64[k] = make_float2((float)cos(a), (float)sin(a));
            }
            SSB_CUDA(ctx, cudaMemcpyToSymbol(kW64, w64, sizeof(w64)));
            std::vector<float2> twm(C64_TWM_ELEMS);
            for (int r = 0; r < 16; ++r)
                for (int tau = 0; tau < 1024; ++tau) {
                    const double a = -2.0 * M_PI * (double)((r * tau) % C64_M) / (double)C64_M;
                    twm[r * 1024 + tau] = make_float2((float)cos(a), (float)sin(a));
                }
            SSB_CUDA(ctx, cudaMalloc(&ctx->twm64, twm.size() * sizeof(float2)));
            SSB_CUDA(ctx, cudaMemcpy(ctx->twm64, twm.data(), twm.size() * sizeof(float2), cudaMemcpyHostToDevice));
            SSB_CUDA(ctx, cudaFuncSetAttribute(conv64k_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C64_SMEM_BYTES));
        }
        SSB_CUDA(ctx, cudaFuncSetAttribute(audio_encoder_conv_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ENC_SMEM_MAX));
        SSB_CUDA(ctx, cudaFuncSetAttribute(audio_encoder_conv_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ENC_SMEM_MAX));
        SSB_CUDA(ctx, cudaFuncSetAttribute(visual_encoder_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ENC_SMEM_MAX));
        SSB_CUDA(ctx, cudaFuncSetAttribute(map_encoder_conv_kernel<8, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, ENC_SMEM_MAX));
        SSB_CUDA(ctx, cudaFuncSetAttribute(map_encoder_conv_kernel<5, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, ENC_SMEM_MAX));
        SSB_CUDA(ctx, cudaFuncSetAttribute(map_encoder_conv_kernel<0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, ENC_SMEM_MAX));
        SSB_CUDA(ctx, cudaFuncSetAttribute(smt_fuse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMT_SMEM_FUSE));
        SSB_CUDA(ctx, cudaFuncSetAttribute(smt_linear_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMT_SMEM_LIN));
        SSB_CUDA(ctx, cudaFuncSetAttribute(smt_attn_kernel,cudaFuncAttributeMaxDynamicSharedMemorySize, SMT_SMEM_ATTN));
        SSB_CUDA(ctx, cudaFuncSetAttribute(smt_enc_tail_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMT_SMEM_TAIL));
        SSB_CUDA(ctx, cudaFuncSetAttribute(smt_decoder_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMT_SMEM_DEC));
        SSB_CUDA(ctx, cudaFuncSetAttribute(smt_dec_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMT_SMEM_DEC_BWD));
        SSB_CUDA(ctx, cudaFuncSetAttribute(smt_enc_tail_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMT_SMEM_TAIL_BWD));
        SSB_CUDA(ctx, cudaFuncSetAttribute(smt_attn_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMT_SMEM_ATTN_BWD));
        SSB_CUDA(ctx, cudaFuncSetAttribute(smt_attn_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMT_SMEM_ATTN_BWD));
        SSB_CUDA(ctx, cudaFuncSetAttribute(smt_fuse_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMT_SMEM_FUSE_BWD));
        SSB_CUDA(ctx, cudaFuncSetAttribute(gru_seq_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GS_SMEM_MAX));
        SSB_CUDA(ctx, cudaFuncSetAttribute(gru_seq_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GS_SMEM_MAX));
        if (setup_smem_attrs<12>() || setup_smem_attrs<13>() || setup_smem_attrs<14>())
            SSB_FAIL(ctx, SSB_E_CUDA, "cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed: %s",
                     cudaGetErrorString(cudaGetLastError()));
        return SSB_OK;
    });
}

extern "C" void ssb_destroy(ssb_ctx* ctx) {
    if (!ctx) return;
    DevGuard guard(ctx->device);
    for (int l = 0; l < 16; ++l)
        if (ctx->tw[l]) cudaFree(ctx->tw[l]);
    if (ctx->window) cudaFree(ctx->window);
    if (ctx->twm64) cudaFree(ctx->twm64);
    if (ctx->yscratch) cudaFree(ctx->yscratch);
    if (ctx->gscratch) cudaFree(ctx->gscratch);
    if (ctx->nscratch) cudaFree(ctx->nscratch);
    if (ctx->head_ticket) cudaFree(ctx->head_ticket);
    if (ctx->s_comp[0]) {
        for (int i = 0; i < SSB_MAX_STREAMS; ++i) { cudaStreamDestroy(ctx->s_comp[i]); cudaEventDestroy(ctx->ev_comp[i]); }
        cudaEventDestroy(ctx->ev_fork);
    }
    if (ctx->s_h2d) {
        cudaStreamDestroy(ctx->s_h2d);
        cudaStreamDestroy(ctx->s_d2h);
        for (int i = 0; i < 2 * SSB_MAX_CHUNKS + 2; ++i)
            if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
        for (int i = 0; i < 2; ++i)
            if (ctx->stage_done[i]) cudaEventDestroy(ctx->stage_done[i]);
    }
    if (ctx->timed) {
        for (auto& tl : *ctx->timed) { cudaEventDestroy(tl.a); cudaEventDestroy(tl.b); }
        delete ctx->timed;
    }
    if (ctx->mel) {
        for (auto& mb : *ctx->mel) { cudaFree(mb.rows); cudaFree(mb.ofs); cudaFree(mb.w); }
        delete ctx->mel;
    }
    for (auto& m : ctx->mstage) {
        if (m.done) cudaEventSynchronize(m.done), cudaEventDestroy(m.done);
        if (m.h) cudaFreeHost(m.h);
        if (m.d) cudaFree(m.d);
    }
    for (auto& r : ctx->rstage) {
        if (r.done) cudaEventSynchronize(r.done), cudaEventDestroy(r.done);
        if (r.h) cudaFreeHost(r.h);
    }
    delete ctx;
}

extern "C" const char* ssb_last_error(const ssb_ctx* ctx) { return ctx ? ctx->err : "null context"; }
extern "C" int64_t ssb_launch_count(const ssb_ctx* ctx) { return ctx ? ctx->launches : 0; }

extern "C" int ssb_set_conv_mode(ssb_ctx* ctx, int mode) {
    if (!ctx || (mode != 0 && mode != 1)) return SSB_E_INVALID_ARG;
    ctx->conv_mode = mode;
    return SSB_OK;
}

extern "C" int ssb_set_streams(ssb_ctx* ctx, int n) {
    if (!ctx || n < 1 || n > SSB_MAX_STREAMS) return SSB_E_INVALID_ARG;
    ctx->n_streams = n;
    return SSB_OK;
}

extern "C" int ssb_set_chunks(ssb_ctx* ctx, int n) {
    if (!ctx || n < 1 || n > 16) return SSB_E_INVALID_ARG;
    ctx->n_chunks = n;
    return SSB_OK;
}

extern "C" int ssb_set_debug(ssb_ctx* ctx, int flags) {
    if (!ctx || (flags & ~32)) return SSB_E_INVALID_ARG;
    ctx->debug = flags;
    return SSB_OK;
}

extern "C" int ssb_set_kernel_timing(ssb_ctx* ctx, int enable) {
    if (!ctx) return SSB_E_INVALID_ARG;
    ctx->timing = enable ? 1 : 0;
    return SSB_OK;
}

extern "C" int ssb_get_kernel_timing(ssb_ctx* ctx, double* ms_sum, int64_t* counts) {
    return abi_call(ctx, [&]() -> int {
        if (!ms_sum || !counts || !ctx->timed) return SSB_E_INVALID_ARG;
        for (int k = 0; k < SSB_N_KERNELS; ++k) { ms_sum[k] = 0.0; counts[k] = 0; }
        for (auto& tl : *ctx->timed) {
            float ms = 0.f;
            cudaError_t e = cudaEventSynchronize(tl.b);
            if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, tl.a, tl.b);
            cudaEventDestroy(tl.a);
            cudaEventDestroy(tl.b);
            if (e != cudaSuccess) { ctx->timed->clear(); SSB_CUDA(ctx, e); }
            ms_sum[tl.kernel] += ms;
            counts[tl.kernel] += 1;
        }
        ctx->timed->clear();
        return SSB_OK;
    });
}

extern "C" int ssb_spec_cols(int sr) {
    const int frames = 1 + sr / SSB_HOP;
    return (frames + SSB_POOL - 1) / SSB_POOL;
}

// The one statement of a valid plan: fills `plan` from (sr, max_taps, n_terms, log2n).  ssb_make_plan returns what it
// makes; check_plan accepts a plan only if this function, given the plan's own fields, makes the same plan again.
static int fill_plan(ssb_ctx* ctx, int sr, int64_t max_taps, int n_terms, int log2n, ssb_plan* plan) {
    if (log2n == C64_LOG2M) {
        // single-block plan: out[m] sits at circular index m + D, D = 65536 - sr; alias-free for taps <= D + 1
        if (n_terms != 1 || sr < SSB_N_FFT || sr > C64_M - C64_NS || max_taps < 0 || max_taps > C64_M - sr + 1)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "single-block plan needs n_terms = 1, sr <= %d and max_taps <= 65536 - sr + 1 "
                     "(sr=%d max_taps=%lld n_terms=%d)", C64_M - C64_NS, sr, (long long)max_taps, n_terms);
        plan->log2n = C64_LOG2M;
        plan->block = C64_M - sr;
        plan->sr = sr;
        plan->n_blocks = 1;
        plan->max_parts = 1;
        plan->n_terms = 1;
        plan->h_elems_per_env = 0;
        return SSB_OK;
    }
    if (log2n < 12 || log2n > 14) SSB_FAIL(ctx, SSB_E_INVALID_ARG, "log2n %d unsupported (12, 13, 14, 16)", log2n);
    if (sr < SSB_N_FFT || max_taps < 0 || n_terms < 1 || n_terms > 2)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "bad plan arguments sr=%d max_taps=%lld n_terms=%d", sr, (long long)max_taps, n_terms);
    const int P = (1 << log2n) / 2;
    plan->log2n = log2n;
    plan->block = P;
    plan->sr = sr;
    plan->n_blocks = (sr + P - 1) / P;
    plan->max_parts = max_taps > 0 ? (int)((max_taps + P - 1) / P) : 1;
    plan->n_terms = n_terms;
    plan->h_elems_per_env = (int64_t)n_terms * plan->max_parts * (1 << log2n);
    return SSB_OK;
}

extern "C" int ssb_make_plan(ssb_ctx* ctx, int sr, int max_taps, int n_terms, int log2n, ssb_plan* plan) {
    if (!ctx || !plan) return SSB_E_INVALID_ARG;
    // default block size: N = 4096 keeps 4 CTAs per SM and the finest tiling; beyond ~12 partitions the per-bin
    // partition sums dominate and N = 8192 is the better plan (at config 3; not re-measured on H100)
    if (log2n == 0) log2n = max_taps > 24576 ? 13 : 12;
    return fill_plan(ctx, sr, max_taps, n_terms, log2n, plan);
}

static_assert(sizeof(ssb_plan) == 6 * sizeof(int32_t) + sizeof(int64_t), "check_plan compares plans byte for byte");

// max_parts * block taps make max_parts partitions again; on the single-block plan (block = 65536 - sr) they are
// within its tap limit
static int check_plan(ssb_ctx* ctx, const ssb_plan* plan) {
    ssb_plan want;
    if (!plan || fill_plan(ctx, plan->sr, (int64_t)plan->max_parts * plan->block, plan->n_terms, plan->log2n, &want) ||
        memcmp(&want, plan, sizeof(want)) != 0)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "invalid plan");
    return SSB_OK;
}

template <int LOG2N>
static cudaError_t launch_src(ssb_ctx* ctx, const float* d_src, int S, int64_t m0, int wrap, int nw, int wofs,
                              float2* d_x, cudaStream_t st) {
    using P = FftPlan<LOG2N>;
    return launch(ctx, SSB_K_FWD_SRC, st, [&] {
        fwd_src_kernel<LOG2N><<<nw, P::T, (P::SMEM_ELEMS + P::TW_SMALL_ELEMS) * sizeof(float2), st>>>(d_src, S, (long long)m0, wrap, wofs, d_x, ctx->tw[LOG2N]);
    });
}

extern "C" int ssb_source_windows(ssb_ctx* ctx, const ssb_plan* plan, const float* d_src, int S, int64_t m0, int wrap,
                                  int nw, int wofs, void* d_x, void* stream) {
    return abi_call(ctx, [&]() -> int {
        int rc = check_plan(ctx, plan);
        if (rc) return rc;
        if (!d_src || !d_x || S <= 0 || nw <= 0 || wofs < 0 || wofs >= nw)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_source_windows: bad arguments (S=%d nw=%d wofs=%d)", S, nw, wofs);
        cudaStream_t st = (cudaStream_t)stream;
        cudaError_t e;
        switch (plan->log2n) {
            case C64_LOG2M:
                if (nw != 1 || wofs != 0) SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_source_windows: the single-block plan has one spectrum (nw = 1, wofs = 0)");
                e = launch(ctx, SSB_K_FWD_SRC, st, [&] {
                    src64k_kernel<<<16, 256, C64_BUF * sizeof(float2), st>>>(d_src, S, (long long)m0, wrap, plan->block, (float2*)d_x,
                                                                            ctx->tw[12], ctx->twm64);
                });
                break;
            case 12: e = launch_src<12>(ctx, d_src, S, m0, wrap, nw, wofs, (float2*)d_x, st); break;
            case 13: e = launch_src<13>(ctx, d_src, S, m0, wrap, nw, wofs, (float2*)d_x, st); break;
            default: e = launch_src<14>(ctx, d_src, S, m0, wrap, nw, wofs, (float2*)d_x, st); break;
        }
        SSB_CUDA(ctx, e);
        return SSB_OK;
    });
}

template <int CL>
static cudaError_t launch_mac_ifft_cluster(ssb_ctx* ctx, const ssb_plan* plan, int B, const ssb_req* d_reqs,
                                           const void* d_xpool, const void* d_h, float* d_wave, int64_t wave_stride,
                                           cudaStream_t st) {
    using P = FftPlan<12>;
    const int lbr = std::min((plan->n_blocks + CL - 1) / CL, (int)kMacRoundBlocks);
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = CL;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(CL * B);
    cfg.blockDim = dim3(P::T);
    cfg.dynamicSmemBytes = (size_t)lbr * P::SMEM_ELEMS * sizeof(float2);
    cfg.stream = st;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    return launch(ctx, SSB_K_MAC_IFFT, st, [&] {   // an error of cudaLaunchKernelEx is also the runtime's last error
        (void)cudaLaunchKernelEx(&cfg, mac_ifft_cluster_kernel<12, CL>, d_reqs, (const float2*)d_xpool, (const float2*)d_h,
                                 plan->max_parts, plan->n_terms, (long long)plan->h_elems_per_env, plan->n_blocks, lbr,
                                 d_wave, (long long)wave_stride, plan->sr, (const float2*)ctx->tw[12]);
    });
}

template <int LOG2N>
static cudaError_t launch_conv_sub(ssb_ctx* ctx, const ssb_plan* plan, int B, const ssb_req* d_reqs, const float* d_rir_bank,
                                   const void* d_xpool, void* d_h, float2* y, float* d_wave, int64_t wave_stride,
                                   cudaStream_t st) {
    using P = FftPlan<LOG2N>;
    const size_t smem = (P::SMEM_ELEMS + P::TW_SMALL_ELEMS) * sizeof(float2);
    cudaError_t e = launch(ctx, SSB_K_FWD_RIR, st, [&] {
        fwd_rir_kernel<LOG2N><<<dim3(plan->max_parts * plan->n_terms, B), P::T, smem, st>>>(
            d_reqs, (const float2*)d_rir_bank, (float2*)d_h, plan->max_parts, (long long)plan->h_elems_per_env, ctx->tw[LOG2N]);
    });
    if (e != cudaSuccess) return e;
    const dim3 g2(B, plan->n_blocks);
    if (ctx->conv_mode == 0) {
        if constexpr (LOG2N == 12) {
            // N = 4096 keeps the partition sums on chip; at N = 8192 and 16384 (512 and 1024 threads per CTA) the
            // cluster kernel held one CTA per SM, or two at 64 registers, and was 5-12 % slower than mac_bins + mac_ifft
            // on config 3 head (DESIGN.md section 5), so those plans keep the sums in Y
            switch (mac_cluster_size(plan->n_blocks)) {
                case 1: return launch_mac_ifft_cluster<1>(ctx, plan, B, d_reqs, d_xpool, d_h, d_wave, wave_stride, st);
                case 2: return launch_mac_ifft_cluster<2>(ctx, plan, B, d_reqs, d_xpool, d_h, d_wave, wave_stride, st);
                case 4: return launch_mac_ifft_cluster<4>(ctx, plan, B, d_reqs, d_xpool, d_h, d_wave, wave_stride, st);
                default: return launch_mac_ifft_cluster<8>(ctx, plan, B, d_reqs, d_xpool, d_h, d_wave, wave_stride, st);
            }
        } else {
            e = launch(ctx, SSB_K_MAC_BINS, st, [&] {
                mac_bins_kernel<LOG2N, 8, 24><<<dim3(P::N / 256, B), 256, 0, st>>>(
                    d_reqs, (const float2*)d_xpool, (const float2*)d_h, plan->max_parts, plan->n_terms,
                    (long long)plan->h_elems_per_env, y, plan->n_blocks, plan->sr);
            });
            if (e != cudaSuccess) return e;
            return launch(ctx, SSB_K_MAC_IFFT, st, [&] {
                mac_ifft_kernel<LOG2N, true><<<g2, P::T, smem, st>>>(d_reqs, (const float2*)d_xpool, y, plan->max_parts,
                                                                     plan->n_terms, (long long)plan->h_elems_per_env, d_wave,
                                                                     (long long)wave_stride, plan->sr, ctx->tw[LOG2N]);
            });
        }
    }
    return launch(ctx, SSB_K_MAC_IFFT, st, [&] {
        mac_ifft_kernel<LOG2N, false><<<g2, P::T, smem, st>>>(d_reqs, (const float2*)d_xpool, (const float2*)d_h, plan->max_parts,
                                                              plan->n_terms, (long long)plan->h_elems_per_env, d_wave,
                                                              (long long)wave_stride, plan->sr, ctx->tw[LOG2N]);
    });
}

// partition-sum scratch Y[B][n_blocks][N] of conv_mode 0 at N >= 8192 (launch_conv_sub), owned by the context
static cudaError_t ensure_yscratch(ssb_ctx* ctx, const ssb_plan* plan, int B) {
    if (ctx->conv_mode != 0 || plan->log2n == 12 || plan->log2n == C64_LOG2M) return cudaSuccess;
    return grow_scratch(ctx->yscratch, ctx->yscratch_elems, (size_t)B * plan->n_blocks * ((size_t)1 << plan->log2n));
}

static cudaError_t launch_conv_any(ssb_ctx* ctx, const ssb_plan* plan, int B, const ssb_req* d_reqs, const float* d_rir_bank,
                                   const void* d_xpool, void* d_h, float2* y, float* d_wave, int64_t wave_stride,
                                   cudaStream_t st) {
    switch (plan->log2n) {
        case C64_LOG2M:
            return launch(ctx, SSB_K_CONV64K, st, [&] {
                conv64k_kernel<<<C64_CL * B, C64_TPB, C64_SMEM_BYTES, st>>>(d_reqs, (const float2*)d_rir_bank, (const float2*)d_xpool,
                                                                            d_wave, (long long)wave_stride, plan->sr, ctx->tw[12], ctx->twm64);
            });
        case 12: return launch_conv_sub<12>(ctx, plan, B, d_reqs, d_rir_bank, d_xpool, d_h, y, d_wave, wave_stride, st);
        case 13: return launch_conv_sub<13>(ctx, plan, B, d_reqs, d_rir_bank, d_xpool, d_h, y, d_wave, wave_stride, st);
        default: return launch_conv_sub<14>(ctx, plan, B, d_reqs, d_rir_bank, d_xpool, d_h, y, d_wave, wave_stride, st);
    }
}

// the refusals of ssb_convolve_batch at B != 0, for a plan check_plan accepted (ssb_render_batch makes them too)
static int check_convolve_args(ssb_ctx* ctx, const ssb_plan* plan, int B, const ssb_req* d_reqs, const float* d_rir_bank,
                               const void* d_xpool, const void* d_hscratch, const float* d_wave, int64_t wave_stride) {
    if (B < 0 || B > 16383 * 4 || !d_reqs || !d_rir_bank || !d_xpool || (!d_hscratch && plan->h_elems_per_env) || !d_wave || wave_stride < plan->sr)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_convolve_batch: bad arguments (B=%d wave_stride=%lld sr=%d)", B,
                 (long long)wave_stride, plan->sr);
    if (((uintptr_t)d_rir_bank & 7) || ((uintptr_t)d_xpool & 7) || ((uintptr_t)d_hscratch & 7))
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_convolve_batch: rir bank / spectra must be 8-byte aligned");
    return SSB_OK;
}

extern "C" int ssb_convolve_batch(ssb_ctx* ctx, const ssb_plan* plan, int B, const ssb_req* d_reqs,
                                  const float* d_rir_bank, const void* d_xpool, void* d_hscratch, float* d_wave,
                                  int64_t wave_stride, void* stream) {
    return abi_call(ctx, [&]() -> int {
        int rc = check_plan(ctx, plan);
        if (rc || B == 0) return rc;
        rc = check_convolve_args(ctx, plan, B, d_reqs, d_rir_bank, d_xpool, d_hscratch, d_wave, wave_stride);
        if (rc) return rc;
        SSB_CUDA(ctx, ensure_yscratch(ctx, plan, B));
        SSB_CUDA(ctx, launch_conv_any(ctx, plan, B, d_reqs, d_rir_bank, d_xpool, d_hscratch, ctx->yscratch, d_wave, wave_stride,
                                      (cudaStream_t)stream));
        return SSB_OK;
    });
}

extern "C" int ssb_crossfade_batch(ssb_ctx* ctx, int B, const float* d_prev, float* d_cur, int sr, int64_t wave_stride,
                                   const uint8_t* d_enable, void* stream) {
    return abi_call(ctx, [&]() -> int {
        if (B == 0) return SSB_OK;
        if (B < 0 || B > 32767 || !d_prev || !d_cur || sr < 20 || wave_stride < sr)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_crossfade_batch: bad arguments");
        const int n_fade = (int)(0.05 * (double)sr);       // int(0.05 * sr), continuous_simulator.py:48
        const dim3 g((n_fade + 1 + 255) / 256, B * 2);
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            crossfade_kernel<<<g, 256, 0, st>>>(d_prev, d_cur, n_fade, (long long)wave_stride, d_enable);
        }));
        return SSB_OK;
    });
}

// the refusals of ssb_spectrogram_batch at B != 0 (ssb_render_batch makes them too)
static int check_spectrogram_args(ssb_ctx* ctx, int B, const float* d_wave, int64_t wave_stride, int sr, int pad_mode,
                                  const float* d_spec) {
    if (B < 0 || B > 65535 || !d_wave || !d_spec || sr < SSB_N_FFT || wave_stride < sr ||
        ((pad_mode & ~SSB_LAYOUT_NCHW) != SSB_PAD_REFLECT && (pad_mode & ~SSB_LAYOUT_NCHW) != SSB_PAD_CONSTANT))
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_spectrogram_batch: bad arguments (B=%d sr=%d pad_mode=%d)", B, sr, pad_mode);
    if (!(pad_mode & SSB_LAYOUT_NCHW) && ((uintptr_t)d_spec & 7))      // the (65, T', 2) layout is stored as float2 (ear pairs)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_spectrogram_batch: d_spec must be 8-byte aligned for the (65, T', 2) layout");
    return SSB_OK;
}

// d_reqs (null: every env is transformed) lets the kernel skip the envs the convolution leaves all zero.
static cudaError_t launch_spectrogram(ssb_ctx* ctx, int B, const float* d_wave, int64_t wave_stride, int sr, int pad_mode,
                                      float* d_spec, const ssb_req* d_reqs, int n_terms, cudaStream_t st) {
    const int nchw = (pad_mode & SSB_LAYOUT_NCHW) ? 1 : 0;
    const int frames = 1 + sr / SSB_HOP;
    const int cols = ssb_spec_cols(sr);
    const dim3 g(cols, B);
    return launch(ctx, SSB_K_SPECTROGRAM, st, [&] {
        if ((pad_mode & ~SSB_LAYOUT_NCHW) == SSB_PAD_REFLECT)
            spectrogram_kernel<true><<<g, 32, 0, st>>>(d_wave, (long long)wave_stride, sr, frames, cols, d_spec, ctx->tw[9],
                                                       ctx->window, nchw, d_reqs, n_terms);
        else
            spectrogram_kernel<false><<<g, 32, 0, st>>>(d_wave, (long long)wave_stride, sr, frames, cols, d_spec, ctx->tw[9],
                                                        ctx->window, nchw, d_reqs, n_terms);
    });
}

extern "C" int ssb_spectrogram_batch(ssb_ctx* ctx, int B, const float* d_wave, int64_t wave_stride, int sr, int pad_mode,
                                     float* d_spec, void* stream) {
    return abi_call(ctx, [&]() -> int {
        if (B == 0) return SSB_OK;
        const int rc = check_spectrogram_args(ctx, B, d_wave, wave_stride, sr, pad_mode, d_spec);
        if (rc) return rc;
        SSB_CUDA(ctx, launch_spectrogram(ctx, B, d_wave, wave_stride, sr, pad_mode, d_spec, nullptr, 0, (cudaStream_t)stream));
        return SSB_OK;
    });
}

// convolve + spectrogram, with every refusal of the two entries decided before the first launch.  With
// ssb_set_streams(ctx, S > 1) the batch is split into S sub-batches whose kernel chains run on S internal streams
// forked from / joined to the caller's stream: the tail of one kernel (partial last wave) overlaps the next
// sub-batch's work, and memory-bound kernels of one chain overlap compute-bound kernels of another.
static int render_batch(ssb_ctx* ctx, const ssb_plan* plan, int B, const ssb_req* d_reqs, const float* d_rir_bank,
                        const void* d_xpool, void* d_hscratch, float* d_wave, int64_t wave_stride, int pad_mode,
                        float* d_spec, void* stream) {
    int rc = check_plan(ctx, plan);
    if (rc || B == 0) return rc;
    rc = check_convolve_args(ctx, plan, B, d_reqs, d_rir_bank, d_xpool, d_hscratch, d_wave, wave_stride);
    if (!rc) rc = check_spectrogram_args(ctx, B, d_wave, wave_stride, plan->sr, pad_mode, d_spec);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    SSB_CUDA(ctx, ensure_yscratch(ctx, plan, B));
    // S streams x C chunks: sub-batch i runs on stream i % S, so a stream works through its chunks one after the
    // other and only S sub-batches' intermediates (H, Y, waveform: 1.3 MB per env at config 2) are live in L2 at a time.
    // One stream (S = 1, also every batch below 64 envs) is the caller's stream itself: one sub-batch, no fork or join.
    const int S = std::max(1, std::min(std::min(ctx->n_streams, SSB_MAX_STREAMS), B / 32));   // sub-batches of at least 32 envs
    int C = S > 1 ? ctx->n_chunks : 1;
    while (C > 1 && B / (S * C) < 16) --C;            // sub-batches of at least 16 envs
    if (S > 1) {
        if (!ctx->s_comp[0]) {
            for (int i = 0; i < SSB_MAX_STREAMS; ++i) {
                SSB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->s_comp[i], cudaStreamNonBlocking));
                SSB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_comp[i], cudaEventDisableTiming));
            }
            SSB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
        }
        SSB_CUDA(ctx, cudaEventRecord(ctx->ev_fork, st));
        for (int i = 0; i < S; ++i) SSB_CUDA(ctx, cudaStreamWaitEvent(ctx->s_comp[i], ctx->ev_fork, 0));
    }
    const size_t spec_row = (size_t)SSB_SPEC_ROWS * ssb_spec_cols(plan->sr) * 2;
    const size_t y_env = (size_t)plan->n_blocks * ((size_t)1 << plan->log2n);
    const int per = (B + S * C - 1) / (S * C);
    int i = 0;
    for (int e0 = 0; e0 < B; e0 += per, ++i) {
        const int nb = std::min(per, B - e0);
        const cudaStream_t si = S > 1 ? ctx->s_comp[i % S] : st;
        float* const wave = d_wave + (size_t)e0 * 2 * wave_stride;
        SSB_CUDA(ctx, launch_conv_any(ctx, plan, nb, d_reqs + e0, d_rir_bank, d_xpool,
                                      (float2*)d_hscratch + (size_t)e0 * plan->h_elems_per_env,
                                      ctx->yscratch ? ctx->yscratch + (size_t)e0 * y_env : nullptr, wave, wave_stride, si));
        SSB_CUDA(ctx, launch_spectrogram(ctx, nb, wave, wave_stride, plan->sr, pad_mode, d_spec + (size_t)e0 * spec_row,
                                         d_reqs + e0, plan->n_terms, si));
    }
    if (S > 1) {
        for (int k = 0; k < S; ++k) {
            SSB_CUDA(ctx, cudaEventRecord(ctx->ev_comp[k], ctx->s_comp[k]));
            SSB_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_comp[k], 0));
        }
    }
    return SSB_OK;
}

extern "C" int ssb_render_batch(ssb_ctx* ctx, const ssb_plan* plan, int B, const ssb_req* d_reqs, const float* d_rir_bank,
                                const void* d_xpool, void* d_hscratch, float* d_wave, int64_t wave_stride, int pad_mode,
                                float* d_spec, void* stream) {
    return abi_call(ctx, [&] {
        return render_batch(ctx, plan, B, d_reqs, d_rir_bank, d_xpool, d_hscratch, d_wave, wave_stride, pad_mode, d_spec, stream);
    });
}

// Host-buffer entry.  n_chunks > 1 pipelines the batch: chunk c+1's H2D copy (copy stream) overlaps
// chunk c's kernels (caller's stream) and chunk c-1's D2H copy (second copy stream); PCIe is full
// duplex, so a step costs about max(H2D, kernels, D2H) instead of their sum.
extern "C" int ssb_render_batch_host(ssb_ctx* ctx, const ssb_plan* plan, int B, const ssb_req* h_reqs, const float* h_rir,
                                     int64_t rir_bytes, float* d_rir_staging, ssb_req* d_reqs_staging, const void* d_xpool,
                                     void* d_hscratch, float* d_wave, int64_t wave_stride, int pad_mode, float* d_spec,
                                     float* h_spec, float* h_wave, int n_chunks, void* stream) {
    return abi_call(ctx, [&]() -> int {
        int rc = check_plan(ctx, plan);
        if (rc) return rc;
        if (B <= 0 || !h_reqs || !h_rir || rir_bytes <= 0 || !d_rir_staging || !d_reqs_staging || !h_spec || !d_spec ||
            !d_wave || wave_stride < plan->sr)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_render_batch_host: bad arguments");
        cudaStream_t st = (cudaStream_t)stream;
        const size_t spec_row = (size_t)SSB_SPEC_ROWS * ssb_spec_cols(plan->sr) * 2;      // floats per env
        if (n_chunks > B) n_chunks = B;
        if (n_chunks > SSB_MAX_CHUNKS) n_chunks = SSB_MAX_CHUNKS;
        if (n_chunks <= 1) {
            SSB_CUDA(ctx, cudaMemcpyAsync(d_rir_staging, h_rir, (size_t)rir_bytes, cudaMemcpyHostToDevice, st));
            SSB_CUDA(ctx, cudaMemcpyAsync(d_reqs_staging, h_reqs, (size_t)B * sizeof(ssb_req), cudaMemcpyHostToDevice, st));
            ctx->last_h2d_bytes = rir_bytes + (int64_t)B * (int64_t)sizeof(ssb_req);
            ctx->last_d2h_bytes = (int64_t)B * (int64_t)spec_row * 4 + (h_wave ? (int64_t)B * 2 * plan->sr * 4 : 0);
            rc = render_batch(ctx, plan, B, d_reqs_staging, d_rir_staging, d_xpool, d_hscratch, d_wave, wave_stride,
                              pad_mode, d_spec, stream);
            if (rc) return rc;
            SSB_CUDA(ctx, cudaMemcpyAsync(h_spec, d_spec, (size_t)B * spec_row * sizeof(float), cudaMemcpyDeviceToHost, st));
            if (h_wave)
                SSB_CUDA(ctx, cudaMemcpy2DAsync(h_wave, (size_t)plan->sr * sizeof(float), d_wave,
                                                (size_t)wave_stride * sizeof(float), (size_t)plan->sr * sizeof(float),
                                                (size_t)B * 2, cudaMemcpyDeviceToHost, st));
            return SSB_OK;
        }
        if (!ctx->s_h2d) {
            SSB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking));
            SSB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking));
            for (int i = 0; i < 2 * SSB_MAX_CHUNKS + 2; ++i)
                SSB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev[i], cudaEventDisableTiming));
            for (int i = 0; i < 2; ++i) SSB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->stage_done[i], cudaEventDisableTiming));
        }
        cudaEvent_t ev_done = ctx->ev[2 * SSB_MAX_CHUNKS + 1];
        // The H2D copies only have to wait for the kernels that last read THIS staging buffer.  A caller
        // that alternates two staging buffers (HostSession does) therefore gets the next step's copy
        // overlapped with the current step's kernels; with a single buffer the copy waits for them.
        for (int i = 0; i < 2; ++i)
            if (ctx->stage_ptr[i] == (const void*)d_rir_staging || ctx->stage_ptr[i] == (const void*)d_reqs_staging)
                SSB_CUDA(ctx, cudaStreamWaitEvent(ctx->s_h2d, ctx->stage_done[i], 0));
        SSB_CUDA(ctx, cudaMemcpyAsync(d_reqs_staging, h_reqs, (size_t)B * sizeof(ssb_req), cudaMemcpyHostToDevice, ctx->s_h2d));
        ctx->last_h2d_bytes = (int64_t)B * (int64_t)sizeof(ssb_req);
        ctx->last_d2h_bytes = (int64_t)B * (int64_t)spec_row * 4 + (h_wave ? (int64_t)B * 2 * plan->sr * 4 : 0);
        const int64_t bank_taps = rir_bytes / (int64_t)sizeof(float2);
        const int per = (B + n_chunks - 1) / n_chunks;
        int c = 0;
        for (int e0 = 0; e0 < B; e0 += per, ++c) {
            const int nb = (B - e0 < per) ? (B - e0) : per;
            // tap ranges of the host bank this chunk reads: silent envs and zero-tap terms need no RIR at all
            // (the reference returns zeros before it even opens the file, simulator.py:610-612); neighbouring
            // ranges are merged so a chunk costs a handful of copies
            std::vector<std::pair<int64_t, int64_t>> runs;
            for (int e = e0; e < e0 + nb; ++e) {
                if (h_reqs[e].flags & SSB_FLAG_SILENT) continue;
                for (int term = 0; term < plan->n_terms; ++term) {
                    const ssb_conv_term& ct = h_reqs[e].term[term];
                    if (ct.rir_taps <= 0) continue;
                    if (ct.rir_offset < 0 || ct.rir_offset + ct.rir_taps > bank_taps)
                        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_render_batch_host: request %d reads outside the host RIR buffer", e);
                    runs.emplace_back(ct.rir_offset, ct.rir_offset + ct.rir_taps);
                }
            }
            std::sort(runs.begin(), runs.end());
            const int64_t kMergeGap = 2048;                         // taps (16 KB): cheaper to copy than to split
            size_t i0 = 0;
            while (i0 < runs.size()) {
                int64_t lo = runs[i0].first, hi = runs[i0].second;
                size_t i1 = i0 + 1;
                while (i1 < runs.size() && runs[i1].first <= hi + kMergeGap) { if (runs[i1].second > hi) hi = runs[i1].second; ++i1; }
                SSB_CUDA(ctx, cudaMemcpyAsync(d_rir_staging + 2 * lo, h_rir + 2 * lo, (size_t)(hi - lo) * sizeof(float2),
                                              cudaMemcpyHostToDevice, ctx->s_h2d));
                ctx->last_h2d_bytes += (hi - lo) * (int64_t)sizeof(float2);
                i0 = i1;
            }
            SSB_CUDA(ctx, cudaEventRecord(ctx->ev[2 * c], ctx->s_h2d));
            SSB_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev[2 * c], 0));
            rc = render_batch(ctx, plan, nb, d_reqs_staging + e0, d_rir_staging, d_xpool,
                              (float2*)d_hscratch + (size_t)e0 * plan->h_elems_per_env, d_wave + (size_t)e0 * 2 * wave_stride,
                              wave_stride, pad_mode, d_spec + (size_t)e0 * spec_row, stream);
            if (rc) return rc;
            SSB_CUDA(ctx, cudaEventRecord(ctx->ev[2 * c + 1], st));
            SSB_CUDA(ctx, cudaStreamWaitEvent(ctx->s_d2h, ctx->ev[2 * c + 1], 0));
            SSB_CUDA(ctx, cudaMemcpyAsync(h_spec + (size_t)e0 * spec_row, d_spec + (size_t)e0 * spec_row,
                                          (size_t)nb * spec_row * sizeof(float), cudaMemcpyDeviceToHost, ctx->s_d2h));
            if (h_wave)
                SSB_CUDA(ctx, cudaMemcpy2DAsync(h_wave + (size_t)e0 * 2 * plan->sr, (size_t)plan->sr * sizeof(float),
                                                d_wave + (size_t)e0 * 2 * wave_stride, (size_t)wave_stride * sizeof(float),
                                                (size_t)plan->sr * sizeof(float), (size_t)nb * 2, cudaMemcpyDeviceToHost,
                                                ctx->s_d2h));
        }
        {   // remember who read this staging buffer last
            const int slot = ctx->stage_next;
            ctx->stage_next ^= 1;
            ctx->stage_ptr[slot] = (const void*)d_rir_staging;
            SSB_CUDA(ctx, cudaEventRecord(ctx->stage_done[slot], st));
        }
        // the caller's stream completes when the last D2H copy has landed
        SSB_CUDA(ctx, cudaEventRecord(ev_done, ctx->s_d2h));
        SSB_CUDA(ctx, cudaStreamWaitEvent(st, ev_done, 0));
        return SSB_OK;
    });
}

extern "C" int ssb_sh_decode_batch(ssb_ctx* ctx, int B, const float* d_amb, int L, const float* d_az_deg, const float* d_hbank,
                                   void* d_filters, float* d_out_rir, void* stream) {
    return abi_call(ctx, [&]() -> int {
        if (B == 0) return SSB_OK;
        if (B < 0 || B > 65535 || L <= 0 || L > SSB_SH_MAX_L)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_sh_decode_batch: bad shape (B=%d L=%d)", B, L);
        if (!d_amb || !d_az_deg || !d_hbank || !d_filters || !d_out_rir || ((uintptr_t)d_amb & 3) || ((uintptr_t)d_az_deg & 3) ||
            ((uintptr_t)d_hbank & 3) || ((uintptr_t)d_filters & 7) || ((uintptr_t)d_out_rir & 7))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_sh_decode_batch: NULL or misaligned pointer");
        cudaStream_t st = (cudaStream_t)stream;
        constexpr int SPAN = SH_TILE + SH_DELAY + SH_TAPS - 1;
        const size_t smem = (size_t)(SH_CH * SPAN + 1) * sizeof(float) + (size_t)SH_CH * SH_TAPS * sizeof(float2);
        if (!ctx->attr_sh) {
            SSB_CUDA(ctx, cudaFuncSetAttribute(sh_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ctx->attr_sh = true;
        }
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { sh_filters_kernel<SH_CH><<<B, SH_TAPS, 0, st>>>(d_hbank, d_az_deg, (float2*)d_filters); }));
        if (L >= 2 * SHF_HOP && !(ctx->debug & 32)) {
            // FFT path: filter spectra (context-owned scratch), then overlap-save blocks
            using P = FftPlan<SHF_LOG2N>;
            SSB_CUDA(ctx, grow_scratch(ctx->gscratch, ctx->gscratch_elems, (size_t)B * SH_CH * P::N));
            const size_t fsmem = (P::SMEM_ELEMS + P::TW_SMALL_ELEMS) * sizeof(float2);
            if (!ctx->attr_shf) {
                SSB_CUDA(ctx, cudaFuncSetAttribute(sh_filter_fft_kernel<SH_CH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
                SSB_CUDA(ctx, cudaFuncSetAttribute(sh_ols_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
                ctx->attr_shf = true;
            }
            SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
                sh_filter_fft_kernel<SH_CH><<<dim3(SH_CH, B), P::T, fsmem, st>>>((const float2*)d_filters, ctx->gscratch, ctx->tw[SHF_LOG2N]);
            }));
            SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
                sh_ols_kernel<<<dim3((L + SHF_HOP - 1) / SHF_HOP, B), P::T, fsmem, st>>>(d_amb, L, ctx->gscratch, d_out_rir,
                                                                                      ctx->tw[SHF_LOG2N]);
            }));
            return SSB_OK;
        }
        const dim3 g((L + SH_TILE - 1) / SH_TILE, B);
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            sh_decode_kernel<<<g, SH_THREADS, smem, st>>>(d_amb, L, (const float2*)d_filters, d_out_rir);
        }));
        return SSB_OK;
    });
}


template <int K>
static cudaError_t sh_multi_set_smem(size_t smem, size_t fsmem) {
    cudaError_t e = cudaFuncSetAttribute(sh_decode_multi_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(sh_filter_fft_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(sh_ols_multi_kernel<K, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(sh_ols_multi_kernel<K, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem);
    return e;
}

template <int K>
static int sh_decode_multi(ssb_ctx* ctx, int n_inputs, int L, const float* d_amb, int n_az, const float* d_az_deg,
                           const float* d_hbank, float2* d_filters, float* d_out, cudaStream_t st) {
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { sh_filters_kernel<K><<<n_az, SH_TAPS, 0, st>>>(d_hbank, d_az_deg, d_filters); }));
    if (L >= 2 * SHF_HOP && !(ctx->debug & 32)) {
        using P = FftPlan<SHF_LOG2N>;
        SSB_CUDA(ctx, grow_scratch(ctx->gscratch, ctx->gscratch_elems, (size_t)n_az * K * P::N));
        const size_t fsmem = (P::SMEM_ELEMS + P::TW_SMALL_ELEMS) * sizeof(float2);
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            sh_filter_fft_kernel<K><<<dim3(K, n_az), P::T, fsmem, st>>>(d_filters, ctx->gscratch, ctx->tw[SHF_LOG2N]);
        }));
        const dim3 g((L + SHF_HOP - 1) / SHF_HOP, n_inputs);
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            if (n_az == 1)
                sh_ols_multi_kernel<K, 1><<<g, P::T, fsmem, st>>>(d_amb, L, n_az, ctx->gscratch, d_out, ctx->tw[SHF_LOG2N]);
            else
                sh_ols_multi_kernel<K, 4><<<g, P::T, fsmem, st>>>(d_amb, L, n_az, ctx->gscratch, d_out, ctx->tw[SHF_LOG2N]);
        }));
        return SSB_OK;
    }
    constexpr int SPAN = SH_TILE + SH_DELAY + SH_TAPS - 1;
    const size_t smem = (size_t)(K * SPAN + 1) * sizeof(float) + (size_t)K * SH_TAPS * sizeof(float2);
    const dim3 g((L + SH_TILE - 1) / SH_TILE, n_inputs);
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        sh_decode_multi_kernel<K><<<g, SH_THREADS, smem, st>>>(d_amb, L, n_az, d_filters, d_out);
    }));
    return SSB_OK;
}

extern "C" int ssb_sh_decode_multi_batch(ssb_ctx* ctx, int n_inputs, int n_channels, int L, const float* d_amb, int n_az,
                                         const float* d_az_deg, const float* d_hbank, void* d_filters, float* d_out,
                                         void* stream) {
    return abi_call(ctx, [&]() -> int {
        const int K = n_channels;
        if (K != 1 && K != 4 && K != 9 && K != 16)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_sh_decode_multi_batch: %d channels (1, 4, 9 or 16: orders 0 to 3)", K);
        if (n_inputs < 0 || n_az < 1 || (long long)n_inputs * n_az > 65535 || L <= 0 || L > SSB_SH_MAX_L)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_sh_decode_multi_batch: bad shape (n_inputs=%d n_az=%d L=%d)", n_inputs, n_az, L);
        if (!d_amb || !d_az_deg || !d_hbank || !d_filters || !d_out || ((uintptr_t)d_amb & 3) || ((uintptr_t)d_az_deg & 3) ||
            ((uintptr_t)d_hbank & 3) || ((uintptr_t)d_filters & 7) || ((uintptr_t)d_out & 7))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_sh_decode_multi_batch: NULL or misaligned pointer");
        if (n_inputs == 0) return SSB_OK;
        // the direct form's input tile and one filter set: 122 KB at K = 16, within the 227 KB a CTA may opt in to
        constexpr int SPAN = SH_TILE + SH_DELAY + SH_TAPS - 1;
        if (!ctx->attr_shm) {
            using P = FftPlan<SHF_LOG2N>;
            const size_t fsmem = (P::SMEM_ELEMS + P::TW_SMALL_ELEMS) * sizeof(float2);
            auto smem = [&](int k) { return (size_t)(k * SPAN + 1) * sizeof(float) + (size_t)k * SH_TAPS * sizeof(float2); };
            SSB_CUDA(ctx, sh_multi_set_smem<1>(smem(1), fsmem));
            SSB_CUDA(ctx, sh_multi_set_smem<4>(smem(4), fsmem));
            SSB_CUDA(ctx, sh_multi_set_smem<9>(smem(9), fsmem));
            SSB_CUDA(ctx, sh_multi_set_smem<16>(smem(16), fsmem));
            ctx->attr_shm = true;
        }
        cudaStream_t st = (cudaStream_t)stream;
        float2* f = (float2*)d_filters;
        switch (K) {
            case 1: return sh_decode_multi<1>(ctx, n_inputs, L, d_amb, n_az, d_az_deg, d_hbank, f, d_out, st);
            case 4: return sh_decode_multi<4>(ctx, n_inputs, L, d_amb, n_az, d_az_deg, d_hbank, f, d_out, st);
            case 9: return sh_decode_multi<9>(ctx, n_inputs, L, d_amb, n_az, d_az_deg, d_hbank, f, d_out, st);
            default: return sh_decode_multi<16>(ctx, n_inputs, L, d_amb, n_az, d_az_deg, d_hbank, f, d_out, st);
        }
    });
}


// ---------------------------------------------------------------------------
// log-mel host side: the Slaney filterbank of librosa.filters.mel(sr, n_fft=512, n_mels, fmin=0, fmax=sr/2,
// htk=False, norm='slaney'), built in double precision, rounded like librosa (float32 triangle, then
// float32(triangle * enorm)) and stored row-sparse.
// ---------------------------------------------------------------------------
static double hz_to_mel_slaney(double f) {
    const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
    return f >= min_log_hz ? min_log_mel + log(f / min_log_hz) / logstep : f / f_sp;
}
static double mel_to_hz_slaney(double m) {
    const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
    return m >= min_log_mel ? min_log_hz * exp(logstep * (m - min_log_mel)) : f_sp * m;
}

// row-sparse filterbank: rows[j] = (first bin, count), ofs[j] = index of the row's first weight in w
static void build_mel_rows(int sr, int n_mels, std::vector<int2>& rows, std::vector<int>& ofs, std::vector<float>& w) {
    const int n_bins = SSB_N_FFT / 2 + 1;
    std::vector<double> mel_f(n_mels + 2);
    const double m_lo = hz_to_mel_slaney(0.0), m_hi = hz_to_mel_slaney(0.5 * (double)sr);
    const double step = (m_hi - m_lo) / (double)(n_mels + 1);
    for (int i = 0; i < n_mels + 2; ++i)        // np.linspace(m_lo, m_hi, n_mels + 2)
        mel_f[i] = mel_to_hz_slaney(i == n_mels + 1 ? m_hi : (double)i * step + m_lo);
    rows.assign(n_mels, make_int2(0, 0));
    ofs.assign(n_mels, 0);
    w.clear();
    std::vector<float> rw(n_bins);
    for (int j = 0; j < n_mels; ++j) {
        const double enorm = 2.0 / (mel_f[j + 2] - mel_f[j]);
        int first = -1, last = -1;
        for (int k = 0; k < n_bins; ++k) {
            const double f = (double)k * ((double)sr / (double)SSB_N_FFT);       // librosa.fft_frequencies(sr, n_fft)
            const double lower = -(mel_f[j] - f) / (mel_f[j + 1] - mel_f[j]);
            const double upper = (mel_f[j + 2] - f) / (mel_f[j + 2] - mel_f[j + 1]);
            const float tri = (float)fmax(0.0, fmin(lower, upper));             // weights[i] is float32 ...
            rw[k] = (float)((double)tri * enorm);                               // ... `weights *= enorm` rounds once more
            if (rw[k] != 0.f) { if (first < 0) first = k; last = k; }
        }
        if (first >= 0) rows[j] = make_int2(first, last - first + 1);
        ofs[j] = (int)w.size();
        for (int k = 0; k < rows[j].y; ++k) w.push_back(rw[rows[j].x + k]);
    }
    if (w.empty()) w.push_back(0.f);
}

// host only (no device needed): dense [n_mels][257] copy of the filterbank the kernels use
extern "C" int ssb_mel_filterbank(int sr, int n_mels, float* h_out) {
    if (sr < SSB_N_FFT || n_mels < 1 || n_mels > MEL_MAX || !h_out) return SSB_E_INVALID_ARG;
    std::vector<int2> rows; std::vector<int> ofs; std::vector<float> w;
    try { build_mel_rows(sr, n_mels, rows, ofs, w); } catch (...) { return SSB_E_OOM; }
    const int n_bins = SSB_N_FFT / 2 + 1;
    for (int j = 0; j < n_mels; ++j) {
        for (int k = 0; k < n_bins; ++k) h_out[j * n_bins + k] = 0.f;
        for (int i = 0; i < rows[j].y; ++i) h_out[j * n_bins + rows[j].x + i] = w[ofs[j] + i];
    }
    return SSB_OK;
}

static int get_mel_bank(ssb_ctx* ctx, int sr, int n_mels, const ssb_ctx::MelBank** out) {
    for (auto& mb : *ctx->mel)
        if (mb.sr == sr && mb.n_mels == n_mels) { *out = &mb; return SSB_OK; }
    std::vector<int2> rows; std::vector<int> ofs; std::vector<float> w;
    build_mel_rows(sr, n_mels, rows, ofs, w);
    ssb_ctx::MelBank mb{sr, n_mels, nullptr, nullptr, nullptr};
    SSB_CUDA(ctx, cudaMalloc(&mb.rows, rows.size() * sizeof(int2)));
    SSB_CUDA(ctx, cudaMalloc(&mb.ofs, ofs.size() * sizeof(int)));
    SSB_CUDA(ctx, cudaMalloc(&mb.w, w.size() * sizeof(float)));
    SSB_CUDA(ctx, cudaMemcpy(mb.rows, rows.data(), rows.size() * sizeof(int2), cudaMemcpyHostToDevice));
    SSB_CUDA(ctx, cudaMemcpy(mb.ofs, ofs.data(), ofs.size() * sizeof(int), cudaMemcpyHostToDevice));
    SSB_CUDA(ctx, cudaMemcpy(mb.w, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice));
    ctx->mel->push_back(mb);
    *out = &ctx->mel->back();
    return SSB_OK;
}

extern "C" int ssb_logmel_frames(int sr) { return 1 + sr / SSB_HOP; }

extern "C" int ssb_logmel_batch(ssb_ctx* ctx, int B, const float* d_wave, int64_t wave_stride, int sr, int n_mels, int power,
                                int pad_mode, float* d_out, void* stream) {
    return abi_call(ctx, [&]() -> int {
        if (B == 0) return SSB_OK;
        if (B < 0 || B > 65535 || !d_wave || !d_out || sr < SSB_N_FFT || wave_stride < sr || n_mels < 1 || n_mels > MEL_MAX ||
            (power != 1 && power != 2) || (pad_mode != SSB_PAD_REFLECT && pad_mode != SSB_PAD_CONSTANT) || ((uintptr_t)d_out & 7))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_logmel_batch: bad arguments (B=%d sr=%d n_mels=%d power=%d pad_mode=%d)", B, sr,
                     n_mels, power, pad_mode);
        const ssb_ctx::MelBank* mb = nullptr;
        const int rc = get_mel_bank(ctx, sr, n_mels, &mb);
        if (rc) return rc;
        const int frames = ssb_logmel_frames(sr);
        const dim3 g((frames + SSB_POOL - 1) / SSB_POOL, B);
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            if (pad_mode == SSB_PAD_REFLECT)
                logmel_kernel<true><<<g, 32, 0, st>>>(d_wave, (long long)wave_stride, sr, frames, n_mels, power, d_out, ctx->tw[9],
                                                       ctx->window, mb->rows, mb->ofs, mb->w);
            else
                logmel_kernel<false><<<g, 32, 0, st>>>(d_wave, (long long)wave_stride, sr, frames, n_mels, power, d_out, ctx->tw[9],
                                                        ctx->window, mb->rows, mb->ofs, mb->w);
        }));
        return SSB_OK;
    });
}

extern "C" int ssb_intensity_batch(ssb_ctx* ctx, int B, const float* d_wave, int64_t wave_stride, int sr, int num_frame,
                                   float* d_out, void* stream) {
    return abi_call(ctx, [&]() -> int {
        if (B == 0) return SSB_OK;
        if (B < 0 || !d_wave || !d_out || sr <= 0 || wave_stride < sr || num_frame <= 0)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_intensity_batch: bad arguments");
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            intensity_kernel<<<B, 256, 0, st>>>(d_wave, (long long)wave_stride, sr, num_frame, d_out);
        }));
        return SSB_OK;
    });
}

extern "C" int ssb_host_copy_bytes(const ssb_ctx* ctx, int64_t* h2d, int64_t* d2h) {
    if (!ctx || !h2d || !d2h) return SSB_E_INVALID_ARG;
    *h2d = ctx->last_h2d_bytes;
    *d2h = ctx->last_d2h_bytes;
    return SSB_OK;
}

extern "C" int ssb_audio_conv1_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W, const float* d_weight,
                                     const float* d_bias, int OC, int KH, int KW, int SH, int SW, int relu, float* d_out,
                                     void* stream) {
    return abi_call(ctx, [&]() -> int {
        if (B == 0) return SSB_OK;
        if (B < 0 || B > 65535 || !d_spec || !d_weight || !d_out || H < 1 || W < 1 || OC < 1 || KH < 1 || KW < 1 || SH < 1 || SW < 1 ||
            KH > H || KW > W)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_audio_conv1_batch: bad arguments (B=%d H=%d W=%d OC=%d K=%dx%d S=%dx%d)", B, H, W, OC, KH,
                     KW, SH, SW);
        const int H1 = (H - KH) / SH + 1, W1 = (W - KW) / SW + 1;
        const size_t smem = ((size_t)KH * W * 2 + (size_t)OC * 2 * KH * KW) * sizeof(float);
        if (W1 * OC > 1024 || smem > 48 * 1024)
            SSB_FAIL(ctx, SSB_E_SHAPE, "ssb_audio_conv1_batch: layer too large for the fused kernel (W1*OC=%d, smem=%zu)", W1 * OC, smem);
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            audio_conv1_kernel<<<dim3(H1, B), W1 * OC, smem, st>>>(d_spec, H, W, d_weight, d_bias, OC, KH, KW, SH, SW, H1, W1,
                                                                  relu, d_out);
        }));
        return SSB_OK;
    });
}

static bool misaligned4(const void* p) { return ((uintptr_t)p & 3u) != 0; }

// ssb_audio_encoder_batch (n_labels = 0, d_labels unused) and ssb_audio_encoder_category_batch; `fn` names the entry
// in error messages
static int audio_encoder(ssb_ctx* ctx, const char* fn, int B, const float* d_spec, int H, int W,
                         const ssb_conv2d_layer* layers, const float* d_labels, int n_labels, int64_t label_stride,
                         const float* d_lin_weight, const float* d_lin_bias, int hidden, int lin_relu,
                         float* d_features, float* d_out, void* stream) {
    if (B < 0 || B > 65535 || !d_spec || misaligned4(d_spec) || !layers || !d_lin_weight || misaligned4(d_lin_weight) ||
        misaligned4(d_lin_bias) || !d_features || misaligned4(d_features) || !d_out || misaligned4(d_out) || H < 1 ||
        W < 1 || hidden < 1 || (lin_relu != 0 && lin_relu != 1))
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d H=%d W=%d hidden=%d lin_relu=%d)", fn, B, H, W, hidden,
                 lin_relu);
    if (n_labels < 0 || (n_labels > 0 && (!d_labels || misaligned4(d_labels))) || label_stride < n_labels)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad labels (n_labels=%d label_stride=%lld d_labels=%p)", fn, n_labels,
                 (long long)label_stride, (const void*)d_labels);
    EncParams p;
    p.H = H;
    p.W = W;
    p.labels = d_labels;
    p.label_stride = label_stride;
    p.n_labels = n_labels;
    int h = H, w = W;
    for (int i = 0; i < 3; ++i) {
        const ssb_conv2d_layer& l = layers[i];
        if (!l.d_weight || misaligned4(l.d_weight) || misaligned4(l.d_bias) || l.out_channels < 1 || l.kh < 1 ||
            l.kw < 1 || l.sh < 1 || l.sw < 1 || (l.relu != 0 && l.relu != 1))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad layer %d (OC=%d K=%dx%d S=%dx%d relu=%d)", fn, i + 1,
                     l.out_channels, l.kh, l.kw, l.sh, l.sw, l.relu);
        if (l.kh > h || l.kw > w)
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: layer %d output is empty (%dx%d input, %dx%d kernel)", fn, i + 1, h, w, l.kh, l.kw);
        h = (h - l.kh) / l.sh + 1;
        w = (w - l.kw) / l.sw + 1;
        p.l[i] = EncLayer{l.d_weight, l.d_bias, l.out_channels, l.kh, l.kw, l.sh, l.sw, l.relu, h, w};
    }
    long long wslice = 0;
    long long ic = 2 + (long long)n_labels;                  // conv1: the two ears, then the label channels
    for (int i = 0; i < 3; ic = p.l[i].oc, ++i)
        wslice = std::max(wslice, enc_wslice(p.l[i].oc, ic, p.l[i].kh * p.l[i].kw));
    const long long smem = ((long long)H * W * 2 + (long long)p.l[0].oc * p.l[0].ho * p.l[0].wo +
                            (long long)p.l[1].oc * p.l[1].ho * p.l[1].wo + wslice) * (long long)sizeof(float);
    if (smem > ENC_SMEM_MAX)
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: observation + conv1 + conv2 activations + weight slice too large for "
                 "the fused kernel (%lld bytes of shared memory > %d)", fn, smem, ENC_SMEM_MAX);
    const long long F = (long long)p.l[2].oc * p.l[2].ho * p.l[2].wo;
    if (F > INT32_MAX) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %lld features", fn, F);
    if (B == 0) return SSB_OK;
    const cudaStream_t st = (cudaStream_t)stream;
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        if (n_labels > 0)
            audio_encoder_conv_kernel<true><<<dim3(ENC_CL, B), ENC_TPB, (size_t)smem, st>>>(d_spec, p, d_features);
        else
            audio_encoder_conv_kernel<false><<<dim3(ENC_CL, B), ENC_TPB, (size_t)smem, st>>>(d_spec, p, d_features);
    }));
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        audio_encoder_linear_kernel<<<dim3((hidden + LIN_ROWS - 1) / LIN_ROWS, (B + LIN_ENVS - 1) / LIN_ENVS), 32 * LIN_WARPS, 0, st>>>(d_features, B, (int)F, d_lin_weight, d_lin_bias, hidden, lin_relu, d_out);
    }));
    return SSB_OK;
}

extern "C" int ssb_audio_encoder_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W, const ssb_conv2d_layer layers[3],
                                       const float* d_lin_weight, const float* d_lin_bias, int hidden, int lin_relu,
                                       float* d_features, float* d_out, void* stream) {
    return abi_call(ctx, [&] { return audio_encoder(ctx, "ssb_audio_encoder_batch", B, d_spec, H, W, layers, nullptr, 0, 0, d_lin_weight, d_lin_bias, hidden, lin_relu, d_features, d_out, stream); });
}

extern "C" int ssb_audio_encoder_category_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W,
                                                const ssb_conv2d_layer layers[3], const float* d_labels, int n_labels,
                                                int64_t label_stride, const float* d_lin_weight, const float* d_lin_bias,
                                                int hidden, int lin_relu, float* d_features, float* d_out, void* stream) {
    return abi_call(ctx, [&] { return audio_encoder(ctx, "ssb_audio_encoder_category_batch", B, d_spec, H, W, layers, d_labels, n_labels, label_stride, d_lin_weight, d_lin_bias, hidden, lin_relu, d_features, d_out, stream); });
}

extern "C" int ssb_visual_encoder_batch(ssb_ctx* ctx, int B, const float* d_rgb, int n_rgb, const float* d_depth,
                                        int n_depth, int H, int W, const ssb_conv2d_layer layers[3],
                                        const float* d_lin_weight, const float* d_lin_bias, int hidden, int lin_relu,
                                        float* d_features, float* d_out, void* stream) {
    static const char* fn = "ssb_visual_encoder_batch";
    return abi_call(ctx, [&]() -> int {
        if (n_rgb < 0 || n_depth < 0)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad channel counts (n_rgb=%d n_depth=%d)", fn, n_rgb, n_depth);
        if (!d_rgb) n_rgb = 0;
        if (!d_depth) n_depth = 0;
        if (B < 0 || B > 65535 || n_rgb + n_depth == 0 || misaligned4(d_rgb) || misaligned4(d_depth) || H < 1 || W < 1 ||
            !layers || !d_lin_weight || misaligned4(d_lin_weight) || misaligned4(d_lin_bias) || hidden < 1 ||
            (lin_relu != 0 && lin_relu != 1) || !d_features || misaligned4(d_features) || !d_out || misaligned4(d_out))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d n_rgb=%d n_depth=%d H=%d W=%d hidden=%d lin_relu=%d)",
                     fn, B, n_rgb, n_depth, H, W, hidden, lin_relu);
        VisParams p;
        p.H = H;
        p.W = W;
        p.n_rgb = n_rgb;
        p.n_depth = n_depth;
        p.rgb = d_rgb;
        p.depth = d_depth;
        int h = H, w = W;
        for (int i = 0; i < 3; ++i) {
            const ssb_conv2d_layer& l = layers[i];
            if (!l.d_weight || misaligned4(l.d_weight) || misaligned4(l.d_bias) || l.out_channels < 1 || l.kh < 1 ||
                l.kw < 1 || l.sh < 1 || l.sw < 1 || (l.relu != 0 && l.relu != 1))
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad layer %d (OC=%d K=%dx%d S=%dx%d relu=%d)", fn, i + 1,
                         l.out_channels, l.kh, l.kw, l.sh, l.sw, l.relu);
            if (l.kh > h || l.kw > w)
                SSB_FAIL(ctx, SSB_E_SHAPE, "%s: layer %d output is empty (%dx%d input, %dx%d kernel)", fn, i + 1, h, w,
                         l.kh, l.kw);
            h = (h - l.kh) / l.sh + 1;
            w = (w - l.kw) / l.sw + 1;
            p.l[i] = EncLayer{l.d_weight, l.d_bias, l.out_channels, l.kh, l.kw, l.sh, l.sw, l.relu, h, w};
        }
        const long long wslice = std::max(enc_wslice(p.l[1].oc, p.l[0].oc, p.l[1].kh * p.l[1].kw),
                                          enc_wslice(p.l[2].oc, p.l[1].oc, p.l[2].kh * p.l[2].kw));
        const long long smem = ((long long)p.l[0].oc * p.l[0].ho * p.l[0].wo + vis_region2(p) + wslice) *
                               (long long)sizeof(float);
        if (smem > ENC_SMEM_MAX)
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: conv1 activations + conv2 activations (or conv1 weights and input rows) + "
                     "weight slice too large for the fused kernel (%lld bytes of shared memory > %d)", fn, smem,
                     ENC_SMEM_MAX);
        const long long F = (long long)p.l[2].oc * p.l[2].ho * p.l[2].wo;
        if (F > INT32_MAX) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %lld features", fn, F);
        if (B == 0) return SSB_OK;
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            visual_encoder_conv_kernel<<<dim3(ENC_CL, B), ENC_TPB, (size_t)smem, st>>>(p, d_features);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            audio_encoder_linear_kernel<<<dim3((hidden + LIN_ROWS - 1) / LIN_ROWS, (B + LIN_ENVS - 1) / LIN_ENVS), 32 * LIN_WARPS, 0, st>>>(d_features, B, (int)F, d_lin_weight, d_lin_bias, hidden, lin_relu, d_out);
        }));
        return SSB_OK;
    });
}

extern "C" int ssb_map_encoder_batch(ssb_ctx* ctx, int B, const float* d_map, int C, int H, int W,
                                     const ssb_conv2d_layer layers[3], const float* d_lin_weight,
                                     const float* d_lin_bias, int hidden, int lin_relu, float* d_features, float* d_out,
                                     void* stream) {
    static const char* fn = "ssb_map_encoder_batch";
    return abi_call(ctx, [&]() -> int {
        if (B < 0 || B > 65535 || C < 1 || H < 1 || W < 1 || !d_map || misaligned4(d_map) || !layers ||
            !d_lin_weight || misaligned4(d_lin_weight) || misaligned4(d_lin_bias) || hidden < 1 ||
            (lin_relu != 0 && lin_relu != 1) || !d_features || misaligned4(d_features) || !d_out || misaligned4(d_out))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d C=%d H=%d W=%d hidden=%d lin_relu=%d)", fn, B, C,
                     H, W, hidden, lin_relu);
        MapParams p;
        p.C = C;
        p.H = H;
        p.W = W;
        p.map = d_map;
        int h = H, w = W;
        for (int i = 0; i < 3; ++i) {
            const ssb_conv2d_layer& l = layers[i];
            if (!l.d_weight || misaligned4(l.d_weight) || misaligned4(l.d_bias) || l.out_channels < 1 || l.kh < 1 ||
                l.kw < 1 || l.sh < 1 || l.sw < 1 || (l.relu != 0 && l.relu != 1))
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad layer %d (OC=%d K=%dx%d S=%dx%d relu=%d)", fn, i + 1,
                         l.out_channels, l.kh, l.kw, l.sh, l.sw, l.relu);
            if (l.kh > h || l.kw > w)
                SSB_FAIL(ctx, SSB_E_SHAPE, "%s: layer %d output is empty (%dx%d input, %dx%d kernel)", fn, i + 1, h, w,
                         l.kh, l.kw);
            h = (h - l.kh) / l.sh + 1;
            w = (w - l.kw) / l.sw + 1;
            p.l[i] = EncLayer{l.d_weight, l.d_bias, l.out_channels, l.kh, l.kw, l.sh, l.sw, l.relu, h, w};
        }
        const double smem = (map_region<double>(p) + map_slice2<double>(p)) * (double)sizeof(float);
        if (smem > ENC_SMEM_MAX)
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: conv1 rows + staged rows and weights + conv2 slice too large for the fused "
                     "kernel (%.0f bytes of shared memory > %d)", fn, smem, ENC_SMEM_MAX);
        const long long F = (long long)p.l[2].oc * p.l[2].ho * p.l[2].wo;
        if (F > INT32_MAX) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %lld features", fn, F);
        if (B == 0) return SSB_OK;
        const cudaStream_t st = (cudaStream_t)stream;
        const EncLayer &L1 = p.l[0], &L2 = p.l[1];
        auto conv = L1.kw == 8 && L2.kh == 4 && L2.kw == 4   ? map_encoder_conv_kernel<8, 4>
                    : L1.kw == 5 && L2.kh == 3 && L2.kw == 3 ? map_encoder_conv_kernel<5, 3>
                                                             : map_encoder_conv_kernel<0, 0>;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            conv<<<dim3(ENC_CL, B), ENC_TPB, (size_t)smem, st>>>(p, d_features);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            audio_encoder_linear_kernel<<<dim3((hidden + LIN_ROWS - 1) / LIN_ROWS, (B + LIN_ENVS - 1) / LIN_ENVS), 32 * LIN_WARPS, 0, st>>>(d_features, B, (int)F, d_lin_weight, d_lin_bias, hidden, lin_relu, d_out);
        }));
        return SSB_OK;
    });
}

extern "C" int ssb_gru_step_batch(ssb_ctx* ctx, int B, int I, int Hd, const float* d_x, const float* d_h,
                                  const float* d_masks, const float* d_w_ih, const float* d_w_hh, const float* d_b_ih,
                                  const float* d_b_hh, float* d_out, float* d_h_out, void* stream) {
    return abi_call(ctx, [&]() -> int {
        const float* ins[] = {d_x, d_h, d_masks, d_w_ih, d_w_hh, d_b_ih, d_b_hh, d_out, d_h_out};
        bool bad = B < 0 || B > 65535 || I < 1 || Hd < 1 || d_out == d_h || d_h_out == d_h;
        for (const float* q : ins) bad = bad || !q || misaligned4(q);
        if (bad)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_gru_step_batch: bad arguments (B=%d I=%d Hd=%d)", B, I, Hd);
        if (B == 0) return SSB_OK;
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            gru_step_kernel<<<dim3(Hd, (B + LIN_ENVS - 1) / LIN_ENVS), 32 * LIN_WARPS, 0, st>>>(
                d_x, d_h, d_masks, B, I, Hd, d_w_ih, d_w_hh, d_b_ih, d_b_hh, d_out, d_h_out);
        }));
        return SSB_OK;
    });
}

static bool gs_overlap(const void* a, size_t na, const void* b, size_t nb) {
    if (!a || !b || !na || !nb) return false;
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + nb && y < x + na;
}

struct GsRange { const void* p; size_t bytes; };

// some output range overlaps an input range or another output range
static bool gs_aliased(const GsRange* outs, int n_outs, const GsRange* ins, int n_ins) {
    for (int i = 0; i < n_outs; ++i) {
        for (int j = 0; j < n_ins; ++j)
            if (gs_overlap(outs[i].p, outs[i].bytes, ins[j].p, ins[j].bytes)) return true;
        for (int j = i + 1; j < n_outs; ++j)
            if (gs_overlap(outs[i].p, outs[i].bytes, outs[j].p, outs[j].bytes)) return true;
    }
    return false;
}

static bool gs_bad_shape(int T, int N, int I, int Hd) {
    return T < 1 || T > SSB_GRU_SEQ_MAX_T || N < 1 || N > SSB_GRU_SEQ_MAX_N || I < 1 || Hd < 1 ||
           Hd > SSB_GRU_SEQ_MAX_HD;
}

extern "C" int64_t ssb_gru_seq_workspace_bytes(int T, int N, int I, int Hd) {
    if (gs_bad_shape(T, N, I, Hd)) return -1;
    return 2LL * T * N * 3 * Hd * (int64_t)sizeof(float);
}

// One CTA per SM at most: U = ceil(Hd / SMs) units per CTA.  Refused (SSB_E_SHAPE) when the W_hh slice does not fit
// or the device cannot hold the grid at once.
static int gs_plan(ssb_ctx* ctx, const char* fn, const void* kernel, int N, int Hd, bool bwd, GruSeqArgs* a,
                   int* grid, size_t* smem) {
    const int U = (Hd + ctx->sm_count - 1) / ctx->sm_count, K = bwd ? 3 * Hd : Hd;
    const int E = std::min(N, std::max(1, GS_STAGE_FLOATS / K));
    *grid = (Hd + U - 1) / U;
    *smem = ((size_t)3 * U * Hd + (size_t)E * K + (bwd ? (size_t)N * U : (size_t)E * 3 * U)) * sizeof(float);
    int occ = 0;
    if (*smem <= (size_t)GS_SMEM_MAX)
        SSB_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, GS_THREADS, *smem));
    if (*smem > (size_t)GS_SMEM_MAX || (long long)occ * ctx->sm_count < *grid)
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %d CTAs of %zu bytes of shared memory do not fit the device at once (%d per SM)",
                 fn, *grid, *smem, occ);
    a->U = U;
    a->E = E;
    return SSB_OK;
}

static cudaError_t gs_launch_coop(ssb_ctx* ctx, cudaStream_t st, const void* kernel, int grid, size_t smem,
                                  GruSeqArgs* a) {
    cudaError_t ce = cudaSuccess;
    const cudaError_t e = launch(ctx, kUntimed, st, [&] {
        void* args[] = {a};
        ce = cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(GS_THREADS), args, smem, st);
    });
    return ce != cudaSuccess ? ce : e;
}

template <bool TA, bool TB>
static cudaError_t gs_gemm(ssb_ctx* ctx, cudaStream_t st, int M, int Nc, int K, const float* A, long long lda,
                           const float* B, long long ldb, const float* bias, float* C, long long ldc, float* rowsum) {
    const dim3 grid(C ? (Nc + GG_BN - 1) / GG_BN : 1, (M + GG_BM - 1) / GG_BM);
    return launch(ctx, kUntimed, st, [&] {
        gru_gemm_kernel<TA, TB><<<grid, GG_THREADS, 0, st>>>(M, Nc, K, A, lda, B, ldb, bias, C, ldc, rowsum);
    });
}

extern "C" int ssb_gru_seq_forward_batch(ssb_ctx* ctx, int T, int N, int I, int Hd, const float* d_x,
                                         const float* d_h0, const float* d_masks, const float* d_w_ih,
                                         const float* d_w_hh, const float* d_b_ih, const float* d_b_hh, float* d_out,
                                         float* d_h_last, float* d_saved, void* d_workspace, void* stream) {
    static const char* fn = "ssb_gru_seq_forward_batch";
    return abi_call(ctx, [&]() -> int {
        const float* need[] = {d_x, d_h0, d_masks, d_w_ih, d_w_hh, d_b_ih, d_b_hh, d_out, d_h_last};
        bool bad = gs_bad_shape(T, N, I, Hd) || misaligned4(d_saved) || !d_workspace || ((uintptr_t)d_workspace & 15u);
        for (const float* q : need) bad = bad || !q || misaligned4(q);
        if (!bad) {
            const size_t TN = (size_t)T * N, f = sizeof(float);
            const GsRange ins[] = {{d_x, TN * I * f}, {d_h0, (size_t)N * Hd * f}, {d_masks, TN * f},
                                   {d_w_ih, 3 * (size_t)Hd * I * f}, {d_w_hh, 3 * (size_t)Hd * Hd * f},
                                   {d_b_ih, 3 * (size_t)Hd * f}, {d_b_hh, 3 * (size_t)Hd * f}};
            const GsRange outs[] = {{d_out, TN * Hd * f}, {d_h_last, (size_t)N * Hd * f}, {d_saved, 5 * TN * Hd * f},
                                    {d_workspace, (size_t)ssb_gru_seq_workspace_bytes(T, N, I, Hd)}};
            bad = gs_aliased(outs, 4, ins, 7);
        }
        if (bad)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (T=%d N=%d I=%d Hd=%d; limits T <= %d, N <= %d, "
                     "Hd <= %d; NULL, misaligned or overlapping buffers refused)", fn, T, N, I, Hd, SSB_GRU_SEQ_MAX_T,
                     SSB_GRU_SEQ_MAX_N, SSB_GRU_SEQ_MAX_HD);
        GruSeqArgs a{};
        int grid = 0;
        size_t smem = 0;
        const int rc = gs_plan(ctx, fn, (const void*)gru_seq_fwd_kernel, N, Hd, false, &a, &grid, &smem);
        if (rc != SSB_OK) return rc;
        float* gi = (float*)d_workspace;
        a.masks = d_masks; a.w_hh = d_w_hh; a.b_hh = d_b_hh; a.h0 = d_h0; a.gi = gi; a.out = d_out;
        a.h_last = d_h_last; a.saved = d_saved; a.T = T; a.N = N; a.Hd = Hd;
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, (gs_gemm<false, true>(ctx, st, T * N, 3 * Hd, I, d_x, I, d_w_ih, I, d_b_ih, gi, 3 * Hd, nullptr)));
        SSB_CUDA(ctx, gs_launch_coop(ctx, st, (const void*)gru_seq_fwd_kernel, grid, smem, &a));
        return SSB_OK;
    });
}

extern "C" int ssb_gru_seq_backward_batch(ssb_ctx* ctx, int T, int N, int I, int Hd, const float* d_x,
                                          const float* d_masks, const float* d_w_ih, const float* d_w_hh,
                                          const float* d_saved, const float* d_grad_out, const float* d_grad_h_last,
                                          void* d_workspace, float* d_dx, float* d_dh0, float* d_dw_ih,
                                          float* d_dw_hh, float* d_db_ih, float* d_db_hh, void* stream) {
    static const char* fn = "ssb_gru_seq_backward_batch";
    return abi_call(ctx, [&]() -> int {
        const float* need[] = {d_x, d_masks, d_w_ih, d_w_hh, d_saved};
        const float* optional[] = {d_grad_out, d_grad_h_last, d_dx, d_dh0, d_dw_ih, d_dw_hh, d_db_ih, d_db_hh};
        bool bad = gs_bad_shape(T, N, I, Hd) || !d_workspace || ((uintptr_t)d_workspace & 15u);
        for (const float* q : need) bad = bad || !q || misaligned4(q);
        for (const float* q : optional) bad = bad || misaligned4(q);
        if (!bad) {
            const size_t TN = (size_t)T * N, f = sizeof(float);
            const GsRange ins[] = {{d_x, TN * I * f}, {d_masks, TN * f}, {d_w_ih, 3 * (size_t)Hd * I * f},
                                   {d_w_hh, 3 * (size_t)Hd * Hd * f}, {d_saved, 5 * TN * Hd * f},
                                   {d_grad_out, TN * Hd * f}, {d_grad_h_last, (size_t)N * Hd * f}};
            const GsRange outs[] = {{d_dx, TN * I * f}, {d_dh0, (size_t)N * Hd * f}, {d_dw_ih, 3 * (size_t)Hd * I * f},
                                    {d_dw_hh, 3 * (size_t)Hd * Hd * f}, {d_db_ih, 3 * (size_t)Hd * f},
                                    {d_db_hh, 3 * (size_t)Hd * f},
                                    {d_workspace, (size_t)ssb_gru_seq_workspace_bytes(T, N, I, Hd)}};
            bad = gs_aliased(outs, 7, ins, 7);
        }
        if (bad)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (T=%d N=%d I=%d Hd=%d; limits T <= %d, N <= %d, "
                     "Hd <= %d; NULL, misaligned or overlapping buffers refused)", fn, T, N, I, Hd, SSB_GRU_SEQ_MAX_T,
                     SSB_GRU_SEQ_MAX_N, SSB_GRU_SEQ_MAX_HD);
        if (!d_dx && !d_dh0 && !d_dw_ih && !d_dw_hh && !d_db_ih && !d_db_hh) return SSB_OK;
        GruSeqArgs a{};
        int grid = 0;
        size_t smem = 0;
        const int rc = gs_plan(ctx, fn, (const void*)gru_seq_bwd_kernel, N, Hd, true, &a, &grid, &smem);
        if (rc != SSB_OK) return rc;
        const long long TN = (long long)T * N, K3 = 3LL * Hd;
        float* dgi = (float*)d_workspace;
        float* dgh = dgi + TN * K3;
        a.masks = d_masks; a.w_hh = d_w_hh; a.saved = (float*)d_saved; a.dout = d_grad_out; a.dh_last = d_grad_h_last;
        a.dgi = dgi; a.dgh = dgh; a.dh0 = d_dh0; a.T = T; a.N = N; a.Hd = Hd;
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, gs_launch_coop(ctx, st, (const void*)gru_seq_bwd_kernel, grid, smem, &a));
        if (d_dx)
            SSB_CUDA(ctx, (gs_gemm<false, false>(ctx, st, (int)TN, I, 3 * Hd, dgi, K3, d_w_ih, I, nullptr, d_dx, I,
                                                 nullptr)));
        if (d_dw_ih || d_db_ih)
            SSB_CUDA(ctx, (gs_gemm<true, false>(ctx, st, 3 * Hd, I, (int)TN, dgi, K3, d_x, I, nullptr, d_dw_ih, I,
                                                d_db_ih)));
        if (d_dw_hh || d_db_hh)
            SSB_CUDA(ctx, (gs_gemm<true, false>(ctx, st, 3 * Hd, Hd, (int)TN, dgh, K3, d_saved, Hd, nullptr, d_dw_hh, Hd,
                                                d_db_hh)));
        return SSB_OK;
    });
}

// The three layers of a conv-stack call, the workspace layout (in floats, each region a multiple of 4) and the
// chunk counts of the weight gradients.
struct CsPlan {
    CsLayer l[3];
    int NL, F;
    long long a1, a2, lb;                          // forward workspace: conv1 and conv2 outputs, label bias
    long long g, dF, da2, da1, part, partb, s;     // backward workspace
    long long fwd_floats, bwd_floats;
    int chunks[3];
};

static long long cs_round4(long long n) { return (n + 3) & ~3LL; }

static int cs_plan(ssb_ctx* ctx, const char* fn, int B, const ssb_conv_stack_input* in, const ssb_conv2d_layer* layers,
                   int lin_in, int hidden, CsPlan* p) {
    if (!in || !layers || B < 0 || B > SSB_CONV_STACK_MAX_B || in->H < 1 || in->W < 1 || hidden < 1 || lin_in < 1)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d hidden=%d in_features=%d; B <= %d)", fn, B, hidden,
                 lin_in, SSB_CONV_STACK_MAX_B);
    const ssb_conv_stack_input& x = *in;
    int nA = 0, nB = 0, kind = 1, scale = 0, NL = 0;
    if (x.kind == SSB_CONV_INPUT_SPECTROGRAM) {
        if (!x.d_x || x.channels != 2 || x.n_labels < 0 || x.n_labels > SSB_CONV_STACK_MAX_LABELS ||
            (x.n_labels > 0 && !x.d_labels) || (x.n_labels > 0 && x.label_stride < x.n_labels))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad spectrogram input (channels=%d n_labels=%d label_stride=%lld)", fn,
                     x.channels, x.n_labels, (long long)x.label_stride);
        nA = 2; kind = 2; NL = x.n_labels;
    } else if (x.kind == SSB_CONV_INPUT_VISUAL) {
        nA = x.d_x ? x.channels : 0;
        nB = x.d_depth ? x.n_depth : 0;
        if (x.channels < 0 || x.n_depth < 0 || nA + nB < 1)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad visual input (n_rgb=%d n_depth=%d)", fn, x.channels, x.n_depth);
        scale = 1;
    } else if (x.kind == SSB_CONV_INPUT_MAP) {
        if (!x.d_x || x.channels < 1)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad map input (channels=%d)", fn, x.channels);
        nA = x.channels;
    } else {
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: unknown input kind %d", fn, x.kind);
    }
    if ((long long)B * x.H * x.W > INT32_MAX)
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %d x %d x %d input pixels exceed 2^31 - 1", fn, B, x.H, x.W);
    int h = x.H, w = x.W, ic = nA + nB;
    for (int i = 0; i < 3; ++i) {
        const ssb_conv2d_layer& l = layers[i];
        if (!l.d_weight || misaligned4(l.d_weight) || misaligned4(l.d_bias) || l.out_channels < 1 || l.kh < 1 ||
            l.kw < 1 || l.sh < 1 || l.sw < 1 || (l.relu != 0 && l.relu != 1))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad layer %d (OC=%d K=%dx%d S=%dx%d relu=%d)", fn, i + 1,
                     l.out_channels, l.kh, l.kw, l.sh, l.sw, l.relu);
        if (l.kh > h || l.kw > w)
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: layer %d output is empty (%dx%d input, %dx%d kernel)", fn, i + 1, h, w, l.kh,
                     l.kw);
        // conv2's and conv3's dX launch one grid z-slice per stride residue class
        if (i > 0 && (long long)l.sh * l.sw > SSB_CONV_STACK_MAX_STRIDE_AREA)
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: layer %d stride %dx%d has more than %d residue classes", fn, i + 1, l.sh,
                     l.sw, SSB_CONV_STACK_MAX_STRIDE_AREA);
        CsLayer& L = p->l[i];
        L = CsLayer{};
        L.kind = i == 0 ? kind : 0;
        L.B = B; L.IC = ic; L.H = h; L.W = w; L.nA = nA; L.nB = nB; L.scale = i == 0 ? scale : 0;
        L.OC = l.out_channels; L.KH = l.kh; L.KW = l.kw; L.SH = l.sh; L.SW = l.sw; L.relu = l.relu;
        L.Ho = (h - l.kh) / l.sh + 1; L.Wo = (w - l.kw) / l.sw + 1;
        L.w = l.d_weight; L.bias = l.d_bias;
        const long long KK = (long long)l.kh * l.kw, K = ic * KK;
        const long long KX = (long long)l.out_channels * ((l.kh + l.sh - 1) / l.sh) * ((l.kw + l.sw - 1) / l.sw);
        const long long outs = (long long)B * l.out_channels * L.Ho * L.Wo;
        if (K > SSB_CONV_STACK_MAX_K || (i > 0 && KX > SSB_CONV_STACK_MAX_K) || outs > INT32_MAX ||
            (long long)B * ic * h * w > INT32_MAX)
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: layer %d: %lld weights per output channel, %lld taps per input channel of its "
                     "transposed conv (each at most %d), %lld outputs (at most 2^31 - 1)", fn, i + 1, K, KX,
                     SSB_CONV_STACK_MAX_K, outs);
        L.K = (int)K;
        L.Kw = (int)((ic + (i == 0 ? NL : 0)) * KK);
        p->chunks[i] = (int)((B * (long long)L.Ho * L.Wo + CS_RCHUNK - 1) / CS_RCHUNK);
        h = L.Ho; w = L.Wo; ic = l.out_channels;
    }
    p->NL = NL;
    const long long F = (long long)ic * h * w;
    if (lin_in != F)
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: Linear in_features %d, conv3 yields %lld features", fn, lin_in, F);
    if ((long long)B * hidden > INT32_MAX)
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: B x hidden = %lld exceeds 2^31 - 1", fn, (long long)B * hidden);
    if (hidden > SSB_CONV_STACK_MAX_HIDDEN)              // the Linear's dW GEMM tiles hidden on grid y, 64 rows a CTA
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: hidden %d exceeds %d", fn, hidden, SSB_CONV_STACK_MAX_HIDDEN);
    p->F = (int)F;
    const CsLayer &L1 = p->l[0], &L2 = p->l[1];
    p->a1 = 0;
    p->a2 = cs_round4((long long)B * L1.OC * L1.Ho * L1.Wo);
    p->lb = p->a2 + cs_round4((long long)B * L2.OC * L2.Ho * L2.Wo);
    p->fwd_floats = p->lb + (NL ? cs_round4((long long)B * L1.OC) : 0);
    long long part = 0, partb = 0;
    for (int i = 0; i < 3; ++i) {
        part = std::max(part, (long long)p->chunks[i] * p->l[i].OC * p->l[i].K);
        partb = std::max(partb, (long long)p->chunks[i] * p->l[i].OC);
    }
    p->g = 0;
    p->dF = cs_round4((long long)B * hidden);
    p->da2 = p->dF + cs_round4((long long)B * F);
    p->da1 = p->da2 + p->a1 + (p->lb - p->a2);
    p->part = p->da1 + p->a2;
    p->partb = p->part + cs_round4(part);
    p->s = p->partb + cs_round4(partb);
    p->bwd_floats = p->s + (NL ? cs_round4((long long)B * L1.OC) : 0);
    return SSB_OK;
}

extern "C" int64_t ssb_conv_stack_train_workspace_bytes(int B, const ssb_conv_stack_input* in,
                                                        const ssb_conv2d_layer layers[3], int lin_in_features,
                                                        int hidden, int backward) {
    CsPlan p;
    if (cs_plan(nullptr, "", B, in, layers, lin_in_features, hidden, &p) != SSB_OK) return -1;
    return (backward ? p.bwd_floats : p.fwd_floats) * (int64_t)sizeof(float);
}

// the caller's input, layer and Linear buffers, for the overlap checks
static int cs_inputs(const CsPlan& p, int B, const ssb_conv_stack_input* in, const ssb_conv2d_layer* layers,
                     const float* lin_w, const float* lin_b, int hidden, GsRange* r) {
    const size_t f = sizeof(float), px = (size_t)B * in->H * in->W;
    int n = 0;
    r[n++] = {in->d_x, px * p.l[0].nA * f};
    r[n++] = {in->kind == SSB_CONV_INPUT_VISUAL ? in->d_depth : nullptr, px * p.l[0].nB * f};
    r[n++] = {p.NL ? in->d_labels : nullptr, B ? ((size_t)(B - 1) * in->label_stride + p.NL) * f : 0};
    for (int i = 0; i < 3; ++i) {
        r[n++] = {layers[i].d_weight, (size_t)p.l[i].OC * p.l[i].Kw * f};
        r[n++] = {layers[i].d_bias, (size_t)p.l[i].OC * f};
    }
    r[n++] = {lin_w, (size_t)hidden * p.F * f};
    r[n++] = {lin_b, (size_t)hidden * f};
    return n;
}

static bool cs_misaligned(const ssb_conv_stack_input* in) {
    return misaligned4(in->d_x) || misaligned4(in->d_depth) || misaligned4(in->d_labels);
}

static cudaError_t cs_launch_gemm(ssb_ctx* ctx, cudaStream_t st, int mode, const CsLayer& L, int chunks) {
    return launch(ctx, kUntimed, st, [&] {
        const size_t smem = (size_t)4 * L.K * sizeof(int);
        if (mode == CS_FWD) {
            const dim3 grid((unsigned)((L.B * (long long)L.Ho * L.Wo + CS_BM - 1) / CS_BM), (L.OC + CS_BN - 1) / CS_BN);
            if (L.kind) cs_gemm_kernel<CS_FWD, true><<<grid, CS_THREADS, smem, st>>>(L);
            else cs_gemm_kernel<CS_FWD, false><<<grid, CS_THREADS, smem, st>>>(L);
        } else if (mode == CS_DW) {
            const dim3 grid(chunks, (L.K + CS_BM - 1) / CS_BM, (L.OC + CS_BN - 1) / CS_BN);
            if (L.kind) cs_gemm_kernel<CS_DW, true><<<grid, CS_THREADS, smem, st>>>(L);
            else cs_gemm_kernel<CS_DW, false><<<grid, CS_THREADS, smem, st>>>(L);
        } else {
            const long long rows = (long long)L.B * ((L.H + L.SH - 1) / L.SH) * ((L.W + L.SW - 1) / L.SW);
            const dim3 grid((unsigned)((rows + CS_BM - 1) / CS_BM), (L.IC + CS_BN - 1) / CS_BN, L.SH * L.SW);
            cs_gemm_kernel<CS_DX, false><<<grid, CS_THREADS, smem, st>>>(L);
        }
    });
}

extern "C" int ssb_conv_stack_train_forward_batch(ssb_ctx* ctx, int B, const ssb_conv_stack_input* in,
                                                  const ssb_conv2d_layer layers[3], const float* d_lin_weight,
                                                  const float* d_lin_bias, int lin_in_features, int hidden,
                                                  int lin_relu, float* d_features, float* d_out, void* d_workspace,
                                                  void* stream) {
    static const char* fn = "ssb_conv_stack_train_forward_batch";
    return abi_call(ctx, [&]() -> int {
        CsPlan p;
        const int rc = cs_plan(ctx, fn, B, in, layers, lin_in_features, hidden, &p);
        if (rc != SSB_OK) return rc;
        bool bad = (lin_relu != 0 && lin_relu != 1) || cs_misaligned(in) || !d_lin_weight ||
                   misaligned4(d_lin_weight) || misaligned4(d_lin_bias) || !d_features || misaligned4(d_features) ||
                   !d_out || misaligned4(d_out) || !d_workspace || ((uintptr_t)d_workspace & 15u);
        if (!bad) {
            GsRange ins[12];
            const int n_ins = cs_inputs(p, B, in, layers, d_lin_weight, d_lin_bias, hidden, ins);
            const size_t f = sizeof(float);
            const GsRange outs[] = {{d_features, (size_t)B * p.F * f}, {d_out, (size_t)B * hidden * f},
                                    {d_workspace, (size_t)p.fwd_floats * f}};
            bad = gs_aliased(outs, 3, ins, n_ins);
        }
        if (bad)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d hidden=%d lin_relu=%d; NULL, misaligned or "
                     "overlapping buffers refused)", fn, B, hidden, lin_relu);
        if (B == 0) return SSB_OK;
        const cudaStream_t st = (cudaStream_t)stream;
        float* ws = (float*)d_workspace;
        CsLayer &L1 = p.l[0], &L2 = p.l[1], &L3 = p.l[2];
        L1.x = in->d_x; L1.x2 = in->d_depth; L1.out = ws + p.a1;
        L2.x = ws + p.a1; L2.out = ws + p.a2;
        L3.x = ws + p.a2; L3.out = d_features;
        if (p.NL) {
            L1.lbias = ws + p.lb;
            SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
                cs_label_bias_kernel<<<(int)(((long long)B * L1.OC + 255) / 256), 256, 0, st>>>(
                    B, L1.OC, p.NL, L1.KH * L1.KW, L1.w, L1.bias, in->d_labels, in->label_stride, ws + p.lb);
            }));
        }
        for (int i = 0; i < 3; ++i) SSB_CUDA(ctx, cs_launch_gemm(ctx, st, CS_FWD, p.l[i], 0));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            audio_encoder_linear_kernel<<<dim3((hidden + LIN_ROWS - 1) / LIN_ROWS, (B + LIN_ENVS - 1) / LIN_ENVS), 32 * LIN_WARPS, 0, st>>>(d_features, B, p.F, d_lin_weight, d_lin_bias, hidden, lin_relu, d_out);
        }));
        return SSB_OK;
    });
}

extern "C" int ssb_conv_stack_train_backward_batch(ssb_ctx* ctx, int B, const ssb_conv_stack_input* in,
                                                   const ssb_conv2d_layer layers[3], const float* d_lin_weight,
                                                   int lin_in_features, int hidden, int lin_relu,
                                                   const float* d_features, const float* d_out, const void* d_saved,
                                                   const float* d_grad_out, void* d_workspace,
                                                   float* const d_grad_weight[4], float* const d_grad_bias[4],
                                                   void* stream) {
    static const char* fn = "ssb_conv_stack_train_backward_batch";
    return abi_call(ctx, [&]() -> int {
        CsPlan p;
        const int rc = cs_plan(ctx, fn, B, in, layers, lin_in_features, hidden, &p);
        if (rc != SSB_OK) return rc;
        bool bad = (lin_relu != 0 && lin_relu != 1) || cs_misaligned(in) || !d_lin_weight ||
                   misaligned4(d_lin_weight) || !d_features || misaligned4(d_features) || !d_out || misaligned4(d_out) ||
                   !d_saved || ((uintptr_t)d_saved & 15u) || !d_grad_out || misaligned4(d_grad_out) || !d_workspace ||
                   ((uintptr_t)d_workspace & 15u) || !d_grad_weight || !d_grad_bias;
        if (!bad) {
            GsRange ins[16];
            int n_ins = cs_inputs(p, B, in, layers, d_lin_weight, nullptr, hidden, ins);
            const size_t f = sizeof(float);
            ins[n_ins++] = {d_features, (size_t)B * p.F * f};
            ins[n_ins++] = {d_out, (size_t)B * hidden * f};
            ins[n_ins++] = {d_saved, (size_t)p.fwd_floats * f};
            ins[n_ins++] = {d_grad_out, (size_t)B * hidden * f};
            GsRange outs[9];
            for (int i = 0; i < 4; ++i) {
                const size_t oc = i < 3 ? (size_t)p.l[i].OC : (size_t)hidden;
                const size_t per = i < 3 ? (size_t)p.l[i].Kw : (size_t)p.F;
                bad = bad || misaligned4(d_grad_weight[i]) || misaligned4(d_grad_bias[i]);
                outs[2 * i] = {d_grad_weight[i], oc * per * f};
                outs[2 * i + 1] = {d_grad_bias[i], oc * f};
            }
            outs[8] = {d_workspace, (size_t)p.bwd_floats * f};
            bad = bad || gs_aliased(outs, 9, ins, n_ins);
        }
        if (bad)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d hidden=%d lin_relu=%d; NULL, misaligned or "
                     "overlapping buffers refused)", fn, B, hidden, lin_relu);
        bool want[4];
        for (int i = 0; i < 4; ++i) want[i] = d_grad_weight[i] || d_grad_bias[i];
        if (B == 0 || !(want[0] || want[1] || want[2] || want[3])) return SSB_OK;
        const cudaStream_t st = (cudaStream_t)stream;
        float* ws = (float*)d_workspace;
        const float* saved = (const float*)d_saved;
        float* g = ws + p.g;
        CsLayer &L1 = p.l[0], &L2 = p.l[1], &L3 = p.l[2];
        L1.x = in->d_x; L1.x2 = in->d_depth;
        L2.x = saved + p.a1; L3.x = saved + p.a2;
        L1.g = ws + p.da1;                          // masked by conv1's ReLU as conv2's dX writes it
        L2.g = ws + p.da2;                          // likewise by conv2's, as conv3's dX writes it
        L3.g = ws + p.dF; L3.gmask = d_features; L3.grelu = L3.relu;
        for (int i = 0; i < 3; ++i) {
            p.l[i].part = ws + p.part;
            p.l[i].partb = ws + p.partb;
        }
        const int n = B * hidden;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            cs_relu_grad_kernel<<<(int)(((long long)n + 255) / 256), 256, 0, st>>>(d_grad_out, d_out, lin_relu, n, g);
        }));
        if (want[3])
            SSB_CUDA(ctx, (gs_gemm<true, false>(ctx, st, hidden, p.F, B, g, hidden, d_features, p.F, nullptr,
                                                d_grad_weight[3], p.F, d_grad_bias[3])));
        const int first = want[0] ? 0 : want[1] ? 1 : want[2] ? 2 : 3;   // the lowest conv whose gradients are needed
        if (first == 3) return SSB_OK;
        SSB_CUDA(ctx, (gs_gemm<false, false>(ctx, st, B, p.F, hidden, g, hidden, d_lin_weight, p.F, nullptr, ws + p.dF,
                                             p.F, nullptr)));
        for (int i = 2; i >= first; --i) {
            CsLayer& L = p.l[i];
            if (want[i]) {
                SSB_CUDA(ctx, cs_launch_gemm(ctx, st, CS_DW, L, p.chunks[i]));
                SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
                    cs_reduce_kernel<<<(L.OC * L.K + L.OC + 255) / 256, 256, 0, st>>>(L, p.chunks[i], d_grad_weight[i],
                                                                                        d_grad_bias[i]);
                }));
                if (i == 0 && p.NL && d_grad_weight[0]) {
                    float* s = ws + p.s;
                    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
                        cs_label_sum_kernel<<<(int)(((long long)B * L.OC + 255) / 256), 256, 0, st>>>(L, s);
                    }));
                    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
                        cs_label_grad_kernel<<<(L.OC * p.NL + 255) / 256, 256, 0, st>>>(
                            B, L.OC, p.NL, L.KH * L.KW, in->d_labels, in->label_stride, s, d_grad_weight[0]);
                    }));
                }
            }
            if (i > first) {                       // dX of this layer's input, the gradient of the layer below
                CsLayer X = L;
                X.out = i == 2 ? ws + p.da2 : ws + p.da1;
                X.xrelu = p.l[i - 1].relu;
                X.K = (int)((long long)L.OC * ((L.KH + L.SH - 1) / L.SH) * ((L.KW + L.SW - 1) / L.SW));
                SSB_CUDA(ctx, cs_launch_gemm(ctx, st, CS_DX, X, 0));
            }
        }
        return SSB_OK;
    });
}

extern "C" int ssb_policy_head_batch(ssb_ctx* ctx, int B, int H, int A, const float* d_features,
                                     const float* d_actor_weight, const float* d_actor_bias,
                                     const float* d_critic_weight, const float* d_critic_bias, int masked,
                                     const float* d_mask, const float* d_q, float* d_value, int64_t* d_action,
                                     float* d_log_prob, float* d_probs, int* d_status, void* stream) {
    static const char* fn = "ssb_policy_head_batch";
    return abi_call(ctx, [&]() -> int {
        const float* need[] = {d_features, d_actor_weight, d_actor_bias, d_critic_weight, d_critic_bias, d_value,
                               d_log_prob};
        const void* optional[] = {d_mask, d_q, d_probs};
        bool bad = B < 0 || B > 65535 || H < 1 || A < 1 || (masked != 0 && masked != 1) || (d_mask && !masked) ||
                   !d_action || ((uintptr_t)d_action & 7u) || !d_status || misaligned4(d_status);
        for (const float* q : need) bad = bad || !q || misaligned4(q);
        for (const void* q : optional) bad = bad || misaligned4(q);
        if (bad)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d H=%d A=%d masked=%d)", fn, B, H, A, masked);
        if (A > PH_MAX_A || H > PH_MAX_H)
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: A=%d H=%d, the kernel is built for A <= %d and H <= %d", fn, A, H,
                     PH_MAX_A, PH_MAX_H);
        if (B == 0) return SSB_OK;
        if (!ctx->head_ticket) {
            SSB_CUDA(ctx, cudaMalloc(&ctx->head_ticket, 2 * sizeof(int)));
            SSB_CUDA(ctx, cudaMemsetAsync(ctx->head_ticket, 0, 2 * sizeof(int), (cudaStream_t)stream));
        }
        const PolicyHeadParams p{d_features, d_actor_weight, d_actor_bias, d_critic_weight, d_critic_bias, d_mask,
                                 d_q, d_value, (long long*)d_action, d_log_prob, d_probs, d_status,
                                 ctx->head_ticket, B, H, A, masked};
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            policy_head_kernel<<<(B + PH_ENVS - 1) / PH_ENVS, 32 * PH_WARPS, 0, st>>>(p);
        }));
        return SSB_OK;
    });
}

static size_t align16(size_t x);

struct PhwLayout {
    size_t dz, partial, tickets, bytes;
    int splits, tiles;
};

static PhwLayout phw_layout(int B, int H, int A) {
    PhwLayout l{};
    l.splits = phw_splits(B);
    l.tiles = ((H + 1 + PHW_TILE - 1) / PHW_TILE) * ((A + 1 + PHW_TILE - 1) / PHW_TILE);
    l.dz = 0;
    l.partial = align16((size_t)B * A * sizeof(float));
    l.tickets = l.partial + align16((size_t)l.splits * (A + 1) * (H + 1) * sizeof(float));
    l.bytes = l.tickets + align16((size_t)l.tiles * sizeof(int));
    return l;
}

extern "C" int64_t ssb_policy_head_train_workspace_bytes(int B, int H, int A) {
    if (B < 0 || B > PH_TRAIN_MAX_B || H < 1 || H > PH_MAX_H || A < 1 || A > PH_MAX_A) return -1;
    return (int64_t)phw_layout(B, H, A).bytes;
}

extern "C" int ssb_policy_head_train_forward_batch(ssb_ctx* ctx, int B, int H, int A, const float* d_features,
                                                   const float* d_actor_weight, const float* d_actor_bias,
                                                   const float* d_critic_weight, const float* d_critic_bias,
                                                   int masked, const float* d_mask, const int64_t* d_action,
                                                   float* d_value, float* d_log_prob, float* d_entropy,
                                                   float* d_saved, int* d_status, void* stream) {
    static const char* fn = "ssb_policy_head_train_forward_batch";
    return abi_call(ctx, [&]() -> int {
        const float* need[] = {d_features, d_actor_weight, d_actor_bias, d_critic_weight, d_critic_bias, d_value,
                               d_log_prob, d_entropy, d_saved};
        bool bad = B < 0 || B > PH_TRAIN_MAX_B || H < 1 || A < 1 || (masked != 0 && masked != 1) ||
                   (d_mask && !masked) || misaligned4(d_mask) || !d_action || ((uintptr_t)d_action & 7u) ||
                   !d_status || misaligned4(d_status);
        for (const float* q : need) bad = bad || !q || misaligned4(q);
        if (bad)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d H=%d A=%d masked=%d)", fn, B, H, A, masked);
        if (A > PH_MAX_A || H > PH_MAX_H)
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: A=%d H=%d, the kernel is built for A <= %d and H <= %d", fn, A, H,
                     PH_MAX_A, PH_MAX_H);
        if (B == 0) return SSB_OK;
        if (!ctx->head_ticket) {
            SSB_CUDA(ctx, cudaMalloc(&ctx->head_ticket, 2 * sizeof(int)));
            SSB_CUDA(ctx, cudaMemsetAsync(ctx->head_ticket, 0, 2 * sizeof(int), (cudaStream_t)stream));
        }
        const PolicyHeadTrainParams p{d_features, d_actor_weight, d_actor_bias, d_critic_weight, d_critic_bias,
                                      d_mask, (const long long*)d_action, d_value, d_log_prob, d_entropy, d_saved,
                                      d_status, ctx->head_ticket, B, H, A, masked};
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            policy_head_train_kernel<<<(B + PH_ENVS - 1) / PH_ENVS, 32 * PH_WARPS, 0, st>>>(p);
        }));
        return SSB_OK;
    });
}

extern "C" int ssb_policy_head_train_backward_batch(ssb_ctx* ctx, int B, int H, int A, const float* d_features,
                                                    const float* d_actor_weight, const float* d_critic_weight,
                                                    int masked, const float* d_mask, const int64_t* d_action,
                                                    const float* d_saved, const float* d_grad_value,
                                                    const float* d_grad_log_prob, const float* d_grad_entropy,
                                                    void* d_workspace, float* d_dfeatures, float* d_dactor_weight,
                                                    float* d_dactor_bias, float* d_dcritic_weight,
                                                    float* d_dcritic_bias, void* stream) {
    static const char* fn = "ssb_policy_head_train_backward_batch";
    return abi_call(ctx, [&]() -> int {
        const float* need[] = {d_features, d_actor_weight, d_critic_weight, d_saved, d_grad_value, d_grad_log_prob,
                               d_grad_entropy};
        const void* optional[] = {d_mask, d_dfeatures, d_dactor_weight, d_dactor_bias, d_dcritic_weight,
                                  d_dcritic_bias};
        bool bad = B < 0 || B > PH_TRAIN_MAX_B || H < 1 || A < 1 || (masked != 0 && masked != 1) ||
                   (d_mask && !masked) || !d_action || ((uintptr_t)d_action & 7u) || !d_workspace ||
                   ((uintptr_t)d_workspace & 15u);
        for (const float* q : need) bad = bad || !q || misaligned4(q);
        for (const void* q : optional) bad = bad || misaligned4(q);
        if (bad)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d H=%d A=%d masked=%d)", fn, B, H, A, masked);
        if (A > PH_MAX_A || H > PH_MAX_H)
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: A=%d H=%d, the kernel is built for A <= %d and H <= %d", fn, A, H,
                     PH_MAX_A, PH_MAX_H);
        const bool params = d_dactor_weight || d_dactor_bias || d_dcritic_weight || d_dcritic_bias;
        if (B == 0 || !(params || d_dfeatures)) return SSB_OK;
        const PhwLayout l = phw_layout(B, H, A);
        char* ws = (char*)d_workspace;
        PolicyHeadBackParams p{d_features, d_actor_weight, d_critic_weight, d_mask, (const long long*)d_action,
                               d_saved, d_grad_value, d_grad_log_prob, d_grad_entropy,
                               params ? (float*)(ws + l.dz) : nullptr, (float*)(ws + l.partial),
                               (int*)(ws + l.tickets), d_dfeatures, d_dactor_weight, d_dactor_bias, d_dcritic_weight,
                               d_dcritic_bias, B, H, A, masked, l.splits, l.tiles};
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            policy_head_dz_kernel<<<(B + PH_WARPS - 1) / PH_WARPS, 32 * PH_WARPS, 0, st>>>(p);
        }));
        if (params) {
            const dim3 grid((H + 1 + PHW_TILE - 1) / PHW_TILE, (A + 1 + PHW_TILE - 1) / PHW_TILE, l.splits);
            SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { policy_head_dw_kernel<<<grid, 256, 0, st>>>(p); }));
        }
        return SSB_OK;
    });
}

// A field of include/ssb200.h into the kernel's form; false when it is outside the limits there.
static bool ro_field(const ssb_rollout_field& in, int n_cols, RoField* out) {
    if (in.T < 1 || in.outer < 1 || in.row_bytes < 1 || in.src_t_stride < 0 || in.src_outer_stride < 0) return false;
    const double bytes = (double)in.outer * in.T * n_cols * (double)in.row_bytes;
    if (bytes >= (double)(1ll << 46)) return false;
    const uintptr_t any = (uintptr_t)in.src | (uintptr_t)in.dst | (uintptr_t)in.row_bytes |
                          (uintptr_t)in.src_t_stride | (uintptr_t)in.src_outer_stride;
    int u = 4;
    while (u > 0 && (any & ((1u << u) - 1))) --u;
    *out = RoField{(const char*)in.src, (char*)in.dst, in.row_bytes, in.src_t_stride, in.src_outer_stride,
                   ((long long)in.outer * in.T * n_cols * in.row_bytes) >> u, in.T, in.outer, u};
    return true;
}

static int ro_fields(ssb_ctx* ctx, const char* fn, const ssb_rollout_field* fields, int n_fields, int n_cols,
                     RoCopyParams* p, long long* units) {
    for (int q = 0; q < n_fields; ++q) {
        if (!fields[q].src || !fields[q].dst)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: field %d has a NULL pointer", fn, q);
        if (!ro_field(fields[q], n_cols, &p->f[q]))
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: field %d (T=%d outer=%d row_bytes=%lld, strides %lld / %lld) is outside "
                     "the limits", fn, q, fields[q].T, fields[q].outer, (long long)fields[q].row_bytes,
                     (long long)fields[q].src_t_stride, (long long)fields[q].src_outer_stride);
        *units += p->f[q].units;
    }
    p->n_fields = n_fields;
    p->n_cols = n_cols;
    return SSB_OK;
}

static int ro_blocks(const ssb_ctx* ctx, long long units) {
    return (int)std::max<long long>(1, std::min<long long>((units + RO_THREADS - 1) / RO_THREADS,
                                                           (long long)ctx->sm_count * 16));
}

extern "C" int ssb_rollout_insert_batch(ssb_ctx* ctx, int N, const ssb_rollout_field* fields, int n_fields,
                                        const ssb_rollout_memory* em, void* stream) {
    static const char* fn = "ssb_rollout_insert_batch";
    return abi_call(ctx, [&]() -> int {
        bool bad = N < 1 || n_fields < 0 || n_fields > SSB_ROLLOUT_MAX_FIELDS || (n_fields > 0 && !fields);
        for (int q = 0; !bad && q < n_fields; ++q)
            bad = (fields[q].on_host != 0 && fields[q].on_host != 1) ||
                  (fields[q].on_host && (fields[q].T != 1 || (fields[q].outer > 1 && fields[q].src_outer_stride)));
        if (em)
            bad = bad || !em->d_masks || misaligned4(em->d_masks) || !em->d_status || misaligned4(em->d_status) ||
                  !em->not_done || misaligned4(em->not_done) || misaligned4(em->d_em_masks_out) ||
                  (em->not_done_on_host != 0 && em->not_done_on_host != 1) || em->total < 1 || em->idx < 0 ||
                  em->idx >= em->total || em->capacity < 0 || em->capacity > em->total || em->step < 0;
        if (bad) SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (N=%d n_fields=%d)", fn, N, n_fields);
        if (N > SSB_ROLLOUT_MAX_ENVS || (em && em->total > SSB_ROLLOUT_MAX_MEMORY))
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: N=%d or a memory of %d slots, the kernel is built for N <= %d and %d slots",
                     fn, N, em ? em->total : 0, SSB_ROLLOUT_MAX_ENVS, SSB_ROLLOUT_MAX_MEMORY);
        ssb_rollout_field local[SSB_ROLLOUT_MAX_FIELDS];
        size_t host_bytes = 0;
        for (int q = 0; q < n_fields; ++q) {
            local[q] = fields[q];
            if (local[q].on_host && local[q].row_bytes > 0) host_bytes += align16((size_t)local[q].row_bytes);
        }
        const bool host_not_done = em && em->not_done_on_host;
        if (host_not_done) host_bytes += align16((size_t)N * sizeof(float));
        const cudaStream_t st = (cudaStream_t)stream;
        ssb_ctx::RolloutStage* stage = nullptr;
        const float* not_done = em ? em->not_done : nullptr;
        if (host_bytes) {
            // Host sources are copied into a pinned, device-mapped ring slot that the kernel reads; the slot is
            // reused once the launch that read it (4 inserts back) has completed.
            for (int q = 0; q < n_fields; ++q)
                if (local[q].on_host && (!local[q].src || local[q].row_bytes < 1))
                    SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: host field %d has a NULL pointer or no bytes", fn, q);
            stage = &ctx->rstage[ctx->rstage_next];
            if (!stage->done) SSB_CUDA(ctx, cudaEventCreateWithFlags(&stage->done, cudaEventDisableTiming));
            SSB_CUDA(ctx, cudaEventSynchronize(stage->done));
            if (host_bytes > stage->cap) {
                if (stage->h) cudaFreeHost(stage->h);
                stage->h = stage->d = nullptr;
                stage->cap = 0;
                const size_t cap = std::max(host_bytes + host_bytes / 4, (size_t)4096);
                SSB_CUDA(ctx, cudaHostAlloc(&stage->h, cap, cudaHostAllocMapped));
                SSB_CUDA(ctx, cudaHostGetDevicePointer(&stage->d, stage->h, 0));
                stage->cap = cap;
            }
            size_t off = 0;
            for (int q = 0; q < n_fields; ++q) {
                if (!local[q].on_host) continue;
                memcpy((char*)stage->h + off, local[q].src, (size_t)local[q].row_bytes);
                local[q].src = (const char*)stage->d + off;
                off += align16((size_t)local[q].row_bytes);
            }
            if (host_not_done) {
                memcpy((char*)stage->h + off, em->not_done, (size_t)N * sizeof(float));
                not_done = (const float*)((const char*)stage->d + off);
            }
        }
        RoCopyParams p;
        long long units = 0;
        if (const int rc = ro_fields(ctx, fn, local, n_fields, 1, &p, &units)) return rc;
        p.has_cols = 0;
        RoMemParams m{};
        int blocks = ro_blocks(ctx, units);
        if (em) {
            m = RoMemParams{em->d_masks, not_done, em->d_em_masks_out, em->d_status, N, em->total, em->capacity,
                            em->idx, em->step};
            blocks = std::max(blocks, N);
        }
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { rollout_insert_kernel<<<blocks, RO_THREADS, 0, st>>>(p, m); }));
        if (stage) {
            SSB_CUDA(ctx, cudaEventRecord(stage->done, st));
            ctx->rstage_next = (ctx->rstage_next + 1) % 4;
        }
        return SSB_OK;
    });
}

extern "C" int ssb_rollout_returns_batch(ssb_ctx* ctx, int N, int S, int T, int scan, int use_gae, float gamma,
                                         float gamma_tau, const float* d_rewards, float* d_value_preds,
                                         float* d_returns, const float* d_masks, const float* d_next_value,
                                         float* d_adv, int normalize, void* stream) {
    static const char* fn = "ssb_rollout_returns_batch";
    return abi_call(ctx, [&]() -> int {
        bool bad = N < 1 || S < 1 || T < 0 || T > S || (scan != 0 && scan != 1) || (use_gae != 0 && use_gae != 1) ||
                   (normalize != 0 && normalize != 1) || (!scan && !d_adv) || !d_value_preds ||
                   misaligned4(d_value_preds) || !d_returns || misaligned4(d_returns) || misaligned4(d_adv);
        if (scan)
            bad = bad || !d_rewards || misaligned4(d_rewards) || !d_masks || misaligned4(d_masks) || !d_next_value ||
                  misaligned4(d_next_value);
        if (bad)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (N=%d S=%d T=%d scan=%d use_gae=%d normalize=%d)", fn,
                     N, S, T, scan, use_gae, normalize);
        if (N > SSB_ROLLOUT_MAX_ENVS || S > SSB_ROLLOUT_MAX_STEPS)
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: N=%d S=%d, the kernel is built for N <= %d and S <= %d", fn, N, S,
                     SSB_ROLLOUT_MAX_ENVS, SSB_ROLLOUT_MAX_STEPS);
        const RoReturnsParams p{d_rewards, d_value_preds, d_returns, d_masks, d_next_value, d_adv, gamma, gamma_tau,
                                N, S, T, scan, use_gae, normalize};
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { rollout_returns_kernel<<<1, RR_THREADS, 0, st>>>(p); }));
        return SSB_OK;
    });
}

extern "C" int ssb_rollout_gather_batch(ssb_ctx* ctx, const ssb_rollout_field* fields, int n_fields, int n_cols,
                                        const int64_t* h_cols, int64_t max_col, void* stream) {
    static const char* fn = "ssb_rollout_gather_batch";
    return abi_call(ctx, [&]() -> int {
        bool host = false;
        for (int q = 0; fields && q < n_fields && q < SSB_ROLLOUT_MAX_FIELDS; ++q) host = host || fields[q].on_host;
        if (n_fields < 1 || n_fields > SSB_ROLLOUT_MAX_FIELDS || !fields || n_cols < 1 || host)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (n_fields=%d n_cols=%d)", fn, n_fields, n_cols);
        if (n_cols > (h_cols ? SSB_ROLLOUT_MAX_COLS : SSB_ROLLOUT_MAX_ENVS))
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %d columns, the kernel is built for %d", fn, n_cols,
                     h_cols ? SSB_ROLLOUT_MAX_COLS : SSB_ROLLOUT_MAX_ENVS);
        RoCopyParams p;
        p.has_cols = h_cols != nullptr;
        for (int j = 0; h_cols && j < n_cols; ++j) {
            if (h_cols[j] < 0 || h_cols[j] >= max_col)
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: column %lld outside [0, %lld)", fn, (long long)h_cols[j],
                         (long long)max_col);
            p.cols[j] = (int)h_cols[j];
        }
        long long units = 0;
        if (const int rc = ro_fields(ctx, fn, fields, n_fields, n_cols, &p, &units)) return rc;
        const int blocks = ro_blocks(ctx, units);
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { rollout_gather_kernel<<<blocks, RO_THREADS, 0, st>>>(p); }));
        return SSB_OK;
    });
}

extern "C" int ssb_belief_update_batch(ssb_ctx* ctx, int B, int num_env, const float* d_spec, int H, int W,
                                       const float* d_pose, int64_t pose_stride, const float* d_loc_pred, int64_t loc_stride,
                                       const float* d_label_pred, int64_t label_stride, const uint8_t* h_dones, double w,
                                       int current_pred_only, float* d_last_pg, uint8_t* d_loc_valid, float* d_last_label,
                                       uint8_t* d_label_valid, float* d_loc_out, float* d_cat_out, void* stream) {
    return abi_call(ctx, [&]() -> int {
        if (B < 0 || num_env < 1 || B > num_env || !d_spec || misaligned4(d_spec) || H < 1 || W < 1 ||
            (current_pred_only != 0 && current_pred_only != 1))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_belief_update_batch: bad arguments (B=%d num_env=%d H=%d W=%d "
                     "current_pred_only=%d)", B, num_env, H, W, current_pred_only);
        if (d_loc_pred && (misaligned4(d_loc_pred) || loc_stride < 2 || !d_pose || misaligned4(d_pose) || pose_stride < 3 ||
                           !d_last_pg || misaligned4(d_last_pg) || !d_loc_valid || !d_loc_out || misaligned4(d_loc_out)))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_belief_update_batch: bad location arguments (loc_stride=%lld pose_stride=%lld)",
                     (long long)loc_stride, (long long)pose_stride);
        if (d_label_pred && (misaligned4(d_label_pred) || label_stride < BELIEF_LABELS || !d_last_label ||
                             misaligned4(d_last_label) || !d_label_valid || !d_cat_out || misaligned4(d_cat_out)))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_belief_update_batch: bad label arguments (label_stride=%lld)",
                     (long long)label_stride);
        if (B > BELIEF_MAX_ENVS)
            SSB_FAIL(ctx, SSB_E_SHAPE, "ssb_belief_update_batch: %d envs > %d (the dones bitmask)", B, BELIEF_MAX_ENVS);
        if (B == 0 || (!d_loc_pred && !d_label_pred)) return SSB_OK;
        BeliefParams p;
        memset(&p, 0, sizeof(p));
        p.spec = d_spec;
        p.spec_len = (long long)H * W * 2;
        p.pose = d_pose;
        p.pose_stride = pose_stride;
        p.loc_pred = d_loc_pred;
        p.loc_stride = loc_stride;
        p.label_pred = d_label_pred;
        p.label_stride = label_stride;
        p.last_pg = d_last_pg;
        p.loc_valid = d_loc_valid;
        p.last_label = d_last_label;
        p.label_valid = d_label_valid;
        p.loc_out = d_loc_out;
        p.cat_out = d_cat_out;
        p.w1 = (float)(1.0 - w);              // numpy rounds a Python float to float32 before it meets a float32 array
        p.w = (float)w;
        p.current_pred_only = current_pred_only;
        p.B = B;
        if (h_dones)
            for (int i = 0; i < B; ++i)
                if (h_dones[i]) p.dones[i >> 5] |= 1u << (i & 31);
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            belief_update_kernel<<<(B + BELIEF_WARPS - 1) / BELIEF_WARPS, 32 * BELIEF_WARPS, 0, st>>>(p);
        }));
        return SSB_OK;
    });
}

// One conv of either ResNet-18 with its geometry and K split.
struct RnLayer { int ic, oc, ks, stride, pad, h, w, ho, wo, tm, S, kps; };

static RnLayer rn_layer(int ic, int oc, int ks, int stride, int pad, int h, int w) {
    RnLayer l{ic, oc, ks, stride, pad, h, w, (h + 2 * pad - ks) / stride + 1, (w + 2 * pad - ks) / stride + 1, 64, 1, 0};
    l.tm = oc <= 16 ? 16 : oc <= 32 ? 32 : 64;
    // K ranges from the layer's shape alone, never from B (an env's sums must not depend on the batch): about 512
    // CTAs at 8 envs, at least 4 K tiles per range
    const int K = ic * ks * ks, kt = (K + RN_TK - 1) / RN_TK, tn = 4096 / l.tm;
    const long long tiles = (long long)((oc + l.tm - 1) / l.tm) * ((8LL * l.ho * l.wo + tn - 1) / tn);
    const int s0 = (int)std::max(1LL, std::min((long long)std::max(1, kt / 4), 512 / tiles));
    l.kps = (kt + s0 - 1) / s0 * RN_TK;
    l.S = (K + l.kps - 1) / l.kps;
    return l;
}

// Geometry of a ResNet-18 on an H x W input with `ic` stem channels, convs in module order: stem, then per block
// conv1, conv2 [, downsample].  Returns the number of features fc takes.
static int rn_geometry(bool smt, int ic, int H, int W, RnLayer* L) {
    static const int kWidthTv[4] = {64, 128, 256, 512}, kWidthSmt[4] = {16, 32, 64, 128};
    const int* width = smt ? kWidthSmt : kWidthTv;
    L[0] = rn_layer(ic, width[0], 7, smt ? 1 : 2, 3, H, W);
    int h = L[0].ho, w = L[0].wo;
    if (!smt) h = (h - 1) / 2 + 1, w = (w - 1) / 2 + 1;       // MaxPool2d(3, 2, 1)
    int n = 1;
    ic = width[0];
    for (int s = 0; s < 4; ++s)
        for (int blk = 0; blk < 2; ++blk) {
            const int stride = s > 0 && blk == 0 ? 2 : 1;
            L[n] = rn_layer(ic, width[s], 3, stride, 1, h, w);
            L[n + 1] = rn_layer(width[s], width[s], 3, 1, 1, L[n].ho, L[n].wo);
            if (stride == 2) L[n + 2] = rn_layer(ic, width[s], 1, 2, 0, h, w);
            h = L[n].ho, w = L[n].wo, ic = width[s];
            n += stride == 2 ? 3 : 2;
        }
    return smt ? width[3] * h * w : width[3];
}

// The eight blocks of either network in module order: the block's conv1 (its conv2 follows it) and its downsample
// conv, or -1; rn_geometry places the convs so.
static const int kRnBlocks[8][2] = {{1, -1}, {3, -1}, {5, 7}, {8, -1}, {10, 12}, {13, -1}, {15, 17}, {18, -1}};

// One network of a ResNet-18 launch sequence: its stem input and layers, parameters, head and scratch.
struct RnNet {
    const float* x;                 // the observation [B][H][W][2] (obs) or an image [B][IC][H][W]
    const ssb_resnet_conv* convs;   // 20, module order
    const float *fc_w, *fc_b;
    int n_out, col;                 // writes out[b][col .. col + n_out)
    const RnLayer* L;               // RN_CONVS layers; all networks of a sequence agree after the stem
    float *A[3], *PA, *PD;          // activations, partial sums of the main convs and of the downsample convs
};

// Scratch floats one network needs at B envs: three activation buffers of `act`, partial sums of `pa` and `pd`.
static size_t rn_scratch(const RnLayer* L, int B, size_t* act, size_t* pa) {
    size_t a = 0, p = 0, d = 0;
    for (int i = 0; i < RN_CONVS; ++i) {
        const size_t out = (size_t)B * L[i].oc * L[i].ho * L[i].wo;
        a = std::max(a, out);
        (L[i].ks == 1 ? d : p) = std::max(L[i].ks == 1 ? d : p, out * L[i].S);
    }
    *act = (a + 3) & ~(size_t)3;
    *pa = (p + 3) & ~(size_t)3;
    return 3 * *act + *pa + ((d + 3) & ~(size_t)3);
}

// Conv i of every network; the stem reads the observation (obs) or each network's image.
static cudaError_t rn_launch_conv(ssb_ctx* ctx, cudaStream_t st, int i, bool obs, int B, int n_in, const RnNet* nets,
                                  const float* const* x, bool downsample, const float* labels, long long label_stride) {
    const RnLayer& l = nets[0].L[i];
    RnConv c{};
    for (int k = 0; k < n_in; ++k) {
        const RnLayer& lk = nets[k].L[i];
        c.in[k] = RnConvIn{nets[k].convs[i].d_weight, x[k], downsample ? nets[k].PD : nets[k].PA, lk.ic,
                           lk.ic * lk.ks * lk.ks, lk.kps};
        c.zs = std::max(c.zs, lk.S);
    }
    c.labels = labels;
    c.label_stride = label_stride;
    c.B = B, c.H = l.h, c.W = l.w, c.OC = l.oc, c.HO = l.ho, c.WO = l.wo, c.stride = l.stride, c.pad = l.pad;
    const long long N = (long long)B * l.ho * l.wo;
    const dim3 grid((unsigned)((N + 4096 / l.tm - 1) / (4096 / l.tm)), (unsigned)((l.oc + l.tm - 1) / l.tm),
                    (unsigned)(n_in * c.zs));
    return launch(ctx, kUntimed, st, [&] {
        if (l.ks == 7 && !obs) rn_conv_kernel<7, false, 16><<<grid, RN_THREADS, 0, st>>>(c);      // SMTCNN stem
        else if (l.ks == 7 && l.tm == 16) rn_conv_kernel<7, true, 16><<<grid, RN_THREADS, 0, st>>>(c);   // SMT stem
        else if (l.ks == 7) rn_conv_kernel<7, true, 64><<<grid, RN_THREADS, 0, st>>>(c);               // torchvision stem
        else if (l.ks == 3 && l.tm == 16) rn_conv_kernel<3, false, 16><<<grid, RN_THREADS, 0, st>>>(c);
        else if (l.ks == 3 && l.tm == 32) rn_conv_kernel<3, false, 32><<<grid, RN_THREADS, 0, st>>>(c);
        else if (l.ks == 3) rn_conv_kernel<3, false, 64><<<grid, RN_THREADS, 0, st>>>(c);
        else if (l.tm == 32) rn_conv_kernel<1, false, 32><<<grid, RN_THREADS, 0, st>>>(c);
        else rn_conv_kernel<1, false, 64><<<grid, RN_THREADS, 0, st>>>(c);
    });
}

// torchvision's stem maxpool on the stem output x of B envs (arg: the window indices, or NULL)
static cudaError_t rn_maxpool(ssb_ctx* ctx, cudaStream_t st, const RnLayer* L, int B, const float* x, float* out,
                              unsigned char* arg) {
    const int hp = L[1].h, wp = L[1].w;
    const long long np = (long long)B * L[0].oc * hp * wp;
    const int blocks = (int)std::min<long long>((np + 255) / 256, (long long)ctx->sm_count * 16);
    return launch(ctx, kUntimed, st, [&] {
        brn_maxpool_kernel<<<blocks, 256, 0, st>>>(x, B * L[0].oc, L[0].ho, L[0].wo, hp, wp, out, arg);
    });
}

// The head of n_in networks on their last block outputs x[k] (avg: the avgpool head, else the flatten head)
static cudaError_t rn_launch_head(ssb_ctx* ctx, cudaStream_t st, int B, int n_in, const RnNet* nets,
                                  const float* const* x, int avg, float* out, int ld) {
    const RnLayer& l = nets[0].L[RN_CONVS - 1];
    RnHead h{};
    for (int k = 0; k < n_in; ++k) h.in[k] = RnHeadIn{x[k], nets[k].fc_w, nets[k].fc_b, nets[k].n_out, nets[k].col};
    h.out = out, h.C = l.oc, h.P = l.ho * l.wo, h.avg = avg, h.ld = ld;
    return launch(ctx, kUntimed, st, [&] { rn_head_kernel<<<dim3(B, n_in), RN_THREADS, 0, st>>>(h); });
}

// The launch sequence of every ResNet-18 forward: the stem, its tail, the blocks in order, the head.  Activation i is
// what finish i writes and -1 the network's input; as a block's input, activation 0 is the stem output after the tail.
// The caller's functors launch conv i on activation `in` (ds: a downsample conv), finish i (with the identity residual
// activation `res` or the downsample conv `ds`, else -1), the stem's tail, and the head on the last block's output.
template <class Conv, class Finish, class Tail, class Head>
static int rn_walk(ssb_ctx* ctx, Conv&& conv, Finish&& finish, Tail&& tail, Head&& head) {
    SSB_CUDA(ctx, conv(0, -1, false));
    SSB_CUDA(ctx, finish(0, -1, -1));
    SSB_CUDA(ctx, tail());
    int x = 0;
    for (const auto& blk : kRnBlocks) {
        const int c1 = blk[0], cd = blk[1];
        SSB_CUDA(ctx, conv(c1, x, false));
        SSB_CUDA(ctx, finish(c1, -1, -1));
        if (cd >= 0) SSB_CUDA(ctx, conv(cd, x, true));
        SSB_CUDA(ctx, conv(c1 + 1, c1, false));
        SSB_CUDA(ctx, finish(c1 + 1, cd >= 0 ? -1 : x, cd));
        x = c1 + 1;
    }
    SSB_CUDA(ctx, head(x));
    return SSB_OK;
}

// Launches every layer of n_in networks side by side (n_in > 1: SMT geometry only), the stem reading the observation
// (obs: [B][H][W][2] plus label channels) or each network's image; the head writes out[b][col ..] with row stride ld.
// smt: GroupNorm(16) and a flatten head, 38 launches; else BatchNorm, maxpool and an avgpool head, 39 launches.
static int rn_forward(ssb_ctx* ctx, cudaStream_t st, bool smt, bool obs, int B, int n_in, const RnNet* nets,
                      const float* labels, long long label_stride, float* out, int ld) {
    const RnLayer* L = nets[0].L;
    // A[slot[i]] holds activation i: A[2] a block's conv1 output (and the torchvision stem's before the maxpool),
    // A[0] and A[1] the block inputs and outputs in turn
    int slot[RN_CONVS] = {smt ? 0 : 2};
    for (int b = 0; b < 8; ++b) slot[kRnBlocks[b][0]] = 2, slot[kRnBlocks[b][0] + 1] = 1 - b % 2;
    auto act = [&](int k, int a) { return a < 0 ? nets[k].x : nets[k].A[a == 0 ? 0 : slot[a]]; };
    auto norm = [&](int k, int i) {
        const ssb_resnet_conv& c = nets[k].convs[i];
        return RnNorm{c.d_gamma, c.d_beta, smt ? nullptr : c.d_mean, smt ? nullptr : c.d_var, c.eps};
    };
    auto conv = [&](int i, int in, bool ds) {
        const float* x[RN_MAX_IN] = {};
        for (int k = 0; k < n_in; ++k) x[k] = act(k, in);
        return rn_launch_conv(ctx, st, i, obs, B, n_in, nets, x, ds, labels, label_stride);
    };
    auto finish = [&](int i, int res, int ds) {
        RnFinish f{};
        for (int k = 0; k < n_in; ++k)
            f.in[k] = RnFinishIn{nets[k].PA, ds >= 0 ? nets[k].PD : nullptr, res >= 0 ? act(k, res) : nullptr,
                                 nets[k].A[slot[i]], norm(k, i), ds >= 0 ? norm(k, ds) : RnNorm{}, nets[k].L[i].S,
                                 ds >= 0 ? nets[k].L[ds].S : 0};
        f.B = B, f.C = L[i].oc, f.P = L[i].ho * L[i].wo, f.relu = 1;
        return launch(ctx, kUntimed, st, [&] { rn_finish_kernel<<<dim3(RN_GROUPS, B, n_in), RN_THREADS, 0, st>>>(f); });
    };
    auto tail = [&] { return smt ? cudaSuccess : rn_maxpool(ctx, st, L, B, nets[0].A[2], nets[0].A[0], nullptr); };
    auto head = [&](int a) {
        const float* x[RN_MAX_IN] = {};
        for (int k = 0; k < n_in; ++k) x[k] = act(k, a);
        return rn_launch_head(ctx, st, B, n_in, nets, x, smt ? 0 : 1, out, ld);
    };
    return rn_walk(ctx, conv, finish, tail, head);
}

// The 20 convs' parameters: non-NULL, aligned, eps > 0, and BatchNorm's running statistics unless smt.
static int rn_check_convs(ssb_ctx* ctx, const char* fn, bool smt, const ssb_resnet_conv* convs, const char* what) {
    for (int i = 0; i < RN_CONVS; ++i) {
        const ssb_resnet_conv& c = convs[i];
        const bool bad_bn = !smt && (!c.d_mean || !c.d_var || misaligned4(c.d_mean) || misaligned4(c.d_var));
        if (!c.d_weight || !c.d_gamma || !c.d_beta || misaligned4(c.d_weight) || misaligned4(c.d_gamma) ||
            misaligned4(c.d_beta) || bad_bn || !(c.eps > 0.f))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad parameters of %sconv %d (eps=%g)", fn, what, i, (double)c.eps);
    }
    return SSB_OK;
}

// ssb_resnet18_batch (smt = false: BatchNorm, maxpool, avgpool head) and ssb_smt_resnet18_batch (smt = true:
// GroupNorm(16), label channels, flatten head); `fn` names the entry in error messages.
static int resnet18(ssb_ctx* ctx, const char* fn, bool smt, int B, const float* d_spec, int H, int W,
                    const float* d_labels, int n_labels, int64_t label_stride, const ssb_resnet_conv* convs,
                    const float* d_fc_weight, const float* d_fc_bias, int fc_in, int n_out, float* d_out, void* stream) {
    if (B < 0 || !d_spec || misaligned4(d_spec) || H < 1 || W < 1 || !convs || !d_fc_weight || misaligned4(d_fc_weight) ||
        misaligned4(d_fc_bias) || fc_in < 1 || n_out < 1 || !d_out || misaligned4(d_out))
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d H=%d W=%d fc_in=%d n_out=%d)", fn, B, H, W, fc_in, n_out);
    if (n_labels < 0 || (n_labels > 0 && (!d_labels || misaligned4(d_labels))) || label_stride < n_labels)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad labels (n_labels=%d label_stride=%lld d_labels=%p)", fn, n_labels,
                 (long long)label_stride, (const void*)d_labels);
    const int rc = rn_check_convs(ctx, fn, smt, convs, "");
    if (rc) return rc;
    if (B > RN_MAX_ENVS) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %d envs > %d", fn, B, RN_MAX_ENVS);
    if (H > RN_MAX_HW || W > RN_MAX_HW) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %dx%d input > %dx%d", fn, H, W, RN_MAX_HW, RN_MAX_HW);
    RnLayer L[RN_CONVS];
    const int feat = rn_geometry(smt, smt ? 2 + n_labels : 2, H, W, L);
    if (fc_in != feat)
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: fc takes %d features; a %dx%d input yields %d", fn, fc_in, H, W, feat);
    if (B == 0) return SSB_OK;
    // scratch: three activation buffers, then the partial sums of a block's main convs and of its downsample conv
    size_t act, pa;
    const size_t need = rn_scratch(L, B, &act, &pa);
    SSB_CUDA(ctx, grow_scratch(ctx->nscratch, ctx->nscratch_elems, (need + 1) / 2));
    float* buf = (float*)ctx->nscratch;
    const RnNet net{d_spec, convs, d_fc_weight, d_fc_bias, n_out, 0, L,
                    {buf, buf + act, buf + 2 * act}, buf + 3 * act, buf + 3 * act + pa};
    return rn_forward(ctx, (cudaStream_t)stream, smt, true, B, 1, &net, d_labels, (long long)label_stride, d_out, n_out);
}

extern "C" int ssb_resnet18_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W, const ssb_resnet_conv convs[20],
                                  const float* d_fc_weight, const float* d_fc_bias, int fc_in, int n_out, float* d_out,
                                  void* stream) {
    return abi_call(ctx, [&] { return resnet18(ctx, "ssb_resnet18_batch", false, B, d_spec, H, W, nullptr, 0, 0, convs, d_fc_weight, d_fc_bias, fc_in, n_out, d_out, stream); });
}

extern "C" int ssb_smt_resnet18_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W, const float* d_labels,
                                      int n_labels, int64_t label_stride, const ssb_resnet_conv convs[20],
                                      const float* d_fc_weight, const float* d_fc_bias, int fc_in, int n_out,
                                      float* d_out, void* stream) {
    return abi_call(ctx, [&] { return resnet18(ctx, "ssb_smt_resnet18_batch", true, B, d_spec, H, W, d_labels, n_labels, label_stride, convs, d_fc_weight, d_fc_bias, fc_in, n_out, d_out, stream); });
}

// The workspace layout, in floats, both networks' ssb_*resnet18_train_* entries share.  The forward keeps, per conv, the
// summed pre-norm values z, the norm's statistics st and the output y of every non-downsample finish (the stem, each
// block's conv1 and its block output).  After those come the network's own saved values, then scratch: the forward's
// K-range partial sums, then (reusing it) the backward's row list, five gradient buffers, dW chunk partials and the
// network's own backward buffers.
struct RnWork {
    RnLayer L[RN_CONVS];
    int feat, rc[RN_CONVS];                             // rc: rows per dW chunk
    long long z[RN_CONVS], st[RN_CONVS], y[RN_CONVS];
    long long live, g[5], part, total;
};

static long long srn_round(long long n) { return (n + 3) & ~3LL; }

// Places z, st (st_floats(l) floats for conv l) and y of every conv from offset off and returns their end; pa and pd
// get the largest K-range partial sums of a main and of a downsample conv.
template <class StFloats>
static long long rn_work_layers(RnWork* w, int B, StFloats st_floats, long long* pa, long long* pd, long long off) {
    *pa = *pd = 0;
    for (int i = 0; i < RN_CONVS; ++i) {
        const RnLayer& l = w->L[i];
        const long long out = (long long)B * l.oc * l.ho * l.wo;
        w->z[i] = off, off += srn_round(out);
        w->st[i] = off, off += srn_round(st_floats(l));
        w->y[i] = -1;
        if (l.ks != 1) w->y[i] = off, off += srn_round(out);
        (l.ks == 1 ? *pd : *pa) = std::max(l.ks == 1 ? *pd : *pa, out * l.S);
    }
    return off;
}

// Places the backward's row list, five gradient buffers and dW chunk partials from off and returns their end.  stem_ic:
// the stem's input channels with a dW GEMM (2 ears of a spectrogram; label channels have none).
static long long rn_work_grads(RnWork* w, int B, long long off, int stem_ic) {
    long long act = 0, part = 0;
    for (int i = 0; i < RN_CONVS; ++i) {
        const RnLayer& l = w->L[i];
        const int P = l.ho * l.wo;
        act = std::max(act, (long long)l.oc * P);
        w->rc[i] = std::max(1, SRN_CHUNK / P);
        const long long K = (long long)(i == 0 ? stem_ic : l.ic) * l.ks * l.ks;
        part = std::max(part, (B + w->rc[i] - 1) / w->rc[i] * (long long)l.oc * K);
    }
    w->live = off, off += srn_round(B + 1LL);                 // B row indices, then the count
    for (int k = 0; k < 5; ++k) w->g[k] = off, off += srn_round((long long)B * act);
    w->part = off, off += srn_round(part);
    return off;
}

// ssb_smt_resnet18_train_*: GroupNorm's (mean, 1 / sqrt(var + eps)) per (row, group) as st; the backward's own
// buffers are the per-row dgamma / dbeta partials and the stem's tap sums.
struct SrnPlan : RnWork {
    int NL, CT, col[RN_CONVS];
    long long pa, pd, gpart, taps;
};

// Lays out one network of geometry p->L and p->NL label channels from offset off (stem_ic as for rn_work_grads); its
// end is p->total.
static void srn_layout(SrnPlan* p, int B, long long off, int stem_ic) {
    long long pa, pd;
    off = rn_work_layers(p, B, [&](const RnLayer&) { return 2LL * B * RN_GROUPS; }, &pa, &pd, off);
    p->CT = 0;
    for (int i = 0; i < RN_CONVS; ++i) p->col[i] = p->CT, p->CT += 2 * p->L[i].oc;
    p->pa = off, p->pd = off + srn_round(pa);
    const long long fwd_end = p->pd + srn_round(pd);
    off = rn_work_grads(p, B, off, stem_ic);
    p->gpart = off, off += srn_round((long long)B * p->CT);
    p->taps = off, off += p->NL ? srn_round((long long)B * p->L[0].oc * 49) : 0;
    p->total = std::max(off, fwd_end);
}

static int srn_plan(ssb_ctx* ctx, const char* fn, int B, int H, int W, int n_labels, int n_out, SrnPlan* p) {
    if (B < 0 || H < 1 || W < 1 || n_labels < 0 || n_out < 1)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d H=%d W=%d n_labels=%d n_out=%d)", fn, B, H, W,
                 n_labels, n_out);
    if (B > SRN_MAX_ENVS) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %d rows > %d", fn, B, SRN_MAX_ENVS);
    if (H > RN_MAX_HW || W > RN_MAX_HW) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %dx%d input > %dx%d", fn, H, W, RN_MAX_HW, RN_MAX_HW);
    p->NL = n_labels;
    p->feat = rn_geometry(true, 2 + n_labels, H, W, p->L);
    srn_layout(p, B, 0, 2);
    return SSB_OK;
}

extern "C" int64_t ssb_smt_resnet18_train_workspace_bytes(int B, int H, int W, int n_labels, int n_out) {
    SrnPlan p;
    if (srn_plan(nullptr, "", B, H, W, n_labels, n_out, &p) != SSB_OK) return -1;
    return p.total * (int64_t)sizeof(float);
}

// What every train entry checks of one network, in this order: the input (named in_name), fc and workspace pointers,
// then `more` (the entry's own arguments), then the 20 convs' parameters (BatchNorm's unless smt; `what` prefixes their
// message).  Then appends the read-only ranges they share: the input (in_bytes), the convs (with the running statistics
// when `stats`) and fc.
template <class More>
static int rn_train_check(ssb_ctx* ctx, const char* fn, bool smt, bool stats, const char* in_name, const float* d_in,
                          size_t in_bytes, const char* what, const ssb_resnet_conv* convs, const float* d_fc_weight,
                          const float* d_fc_bias, int fc_in, int n_out, const void* d_workspace, const RnLayer* L,
                          More&& more, GsRange* ins, int* n_ins) {
    if (!d_in || misaligned4(d_in) || !convs || !d_fc_weight || misaligned4(d_fc_weight) || misaligned4(d_fc_bias) ||
        !d_workspace || ((uintptr_t)d_workspace & 15u))
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (NULL or misaligned %s, fc or workspace)", fn, in_name);
    const int rc = more();
    if (rc) return rc;
    const int rcv = rn_check_convs(ctx, fn, smt, convs, what);
    if (rcv) return rcv;
    const size_t f = sizeof(float);
    int n = *n_ins;
    ins[n++] = {d_in, in_bytes};
    for (int i = 0; i < RN_CONVS; ++i) {
        const RnLayer& l = L[i];
        ins[n++] = {convs[i].d_weight, (size_t)l.oc * l.ic * l.ks * l.ks * f};
        ins[n++] = {convs[i].d_gamma, (size_t)l.oc * f};
        ins[n++] = {convs[i].d_beta, (size_t)l.oc * f};
        if (stats) {
            ins[n++] = {convs[i].d_mean, (size_t)l.oc * f};
            ins[n++] = {convs[i].d_var, (size_t)l.oc * f};
        }
    }
    ins[n++] = {d_fc_weight, (size_t)n_out * fc_in * f};
    ins[n++] = {d_fc_bias, (size_t)n_out * f};
    *n_ins = n;
    return SSB_OK;
}

// the arguments both train entries share: shape, labels, parameters and fc; then the caller's read-only buffers
static int srn_check(ssb_ctx* ctx, const char* fn, int B, const float* d_spec, int H, int W, const float* d_labels,
                     int n_labels, int64_t label_stride, const ssb_resnet_conv* convs, const float* d_fc_weight,
                     const float* d_fc_bias, int fc_in, int n_out, const void* d_workspace, SrnPlan* p, GsRange* ins,
                     int* n_ins) {
    int rc = srn_plan(ctx, fn, B, H, W, n_labels, n_out, p);
    if (rc != SSB_OK) return rc;
    rc = rn_train_check(ctx, fn, true, false, "spectrogram", d_spec, (size_t)B * H * W * 2 * sizeof(float), "", convs,
                        d_fc_weight, d_fc_bias, fc_in, n_out, d_workspace, p->L, [&]() -> int {
        if ((n_labels > 0 && (!d_labels || misaligned4(d_labels))) || label_stride < n_labels)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad labels (n_labels=%d label_stride=%lld d_labels=%p)", fn, n_labels,
                     (long long)label_stride, (const void*)d_labels);
        return SSB_OK;
    }, ins, n_ins);
    if (rc != SSB_OK) return rc;
    if (fc_in != p->feat)
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: fc takes %d features; a %dx%d input yields %d", fn, fc_in, H, W, p->feat);
    ins[(*n_ins)++] = {n_labels ? d_labels : nullptr, B ? ((size_t)(B - 1) * label_stride + n_labels) * sizeof(float) : 0};
    return SSB_OK;
}

// The backward entries' gradient outputs of one network: the arrays non-NULL, every gradient aligned, and none of them
// or the workspace overlapping another or a read-only range (ins, to which d_dpred, row stride ld, is added).  On
// success the gradients are appended to ins too (room for 2 + 3 RN_CONVS more), so that the next network's check
// refuses gradients that overlap these.
static int rn_check_grads(ssb_ctx* ctx, const char* fn, const RnWork& p, int B, int fc_in, int n_out, int ld,
                          const float* d_dpred, const void* d_workspace, float* const* d_dweight,
                          float* const* d_dgamma, float* const* d_dbeta, const float* d_dfc_weight,
                          const float* d_dfc_bias, GsRange* ins, int* n_ins) {
    const size_t f = sizeof(float);
    ins[(*n_ins)++] = {d_dpred, B ? ((size_t)(B - 1) * ld + n_out) * f : 0};
    bool bad = !d_dpred || misaligned4(d_dpred) || !d_dweight || !d_dgamma || !d_dbeta || misaligned4(d_dfc_weight) ||
               misaligned4(d_dfc_bias);
    GsRange outs[3 + 3 * RN_CONVS];
    int n_outs = 0;
    if (!bad) {
        for (int i = 0; i < RN_CONVS; ++i) {
            const RnLayer& l = p.L[i];
            bad = bad || misaligned4(d_dweight[i]) || misaligned4(d_dgamma[i]) || misaligned4(d_dbeta[i]);
            outs[n_outs++] = {d_dweight[i], (size_t)l.oc * l.ic * l.ks * l.ks * f};
            outs[n_outs++] = {d_dgamma[i], (size_t)l.oc * f};
            outs[n_outs++] = {d_dbeta[i], (size_t)l.oc * f};
        }
        outs[n_outs++] = {d_dfc_weight, (size_t)n_out * fc_in * f};
        outs[n_outs++] = {d_dfc_bias, (size_t)n_out * f};
        outs[n_outs++] = {d_workspace, (size_t)p.total * f};
        bad = bad || gs_aliased(outs, n_outs, ins, *n_ins);
    }
    if (bad)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad gradient arguments (NULL, misaligned or overlapping buffers "
                 "refused)", fn);
    for (int i = 0; i + 1 < n_outs; ++i) ins[(*n_ins)++] = outs[i];
    return SSB_OK;
}

// The GroupNorm training forward of one network (net: stem input, parameters, head columns) on the workspace ws of
// layout p: rn_forward's launches with a buffer per layer and the saving finish, so the same K splits and bits.  The
// stem reads net.x as the observation plus label channels (obs) or as an image; the head writes out[b][net.col ..]
// with row stride ld.  38 launches.
static int srn_forward(ssb_ctx* ctx, cudaStream_t st, const SrnPlan& p, float* ws, int B, const RnNet& net, bool obs,
                       const float* labels, long long label_stride, float* out, int ld) {
    const RnLayer* L = p.L;
    const ssb_resnet_conv* convs = net.convs;
    RnNet n = net;
    n.L = L, n.PA = ws + p.pa, n.PD = ws + p.pd;
    auto act = [&](int a) -> const float* { return a < 0 ? n.x : ws + p.y[a]; };
    auto norm = [&](int i) { return RnNorm{convs[i].d_gamma, convs[i].d_beta, nullptr, nullptr, convs[i].eps}; };
    auto conv = [&](int i, int in, bool ds) {
        const float* xs[RN_MAX_IN] = {act(in)};
        return rn_launch_conv(ctx, st, i, obs && i == 0, B, 1, &n, xs, ds, labels, label_stride);
    };
    auto finish = [&](int i, int res, int ds) {
        RnFinish f{};
        f.in[0] = RnFinishIn{n.PA, ds >= 0 ? n.PD : nullptr, res >= 0 ? act(res) : nullptr, ws + p.y[i],
                             norm(i), ds >= 0 ? norm(ds) : RnNorm{}, L[i].S, ds >= 0 ? L[ds].S : 0};
        f.B = B, f.C = L[i].oc, f.P = L[i].ho * L[i].wo, f.relu = 1;
        const RnSave s{ws + p.z[i], ds >= 0 ? ws + p.z[ds] : nullptr, (float2*)(ws + p.st[i]),
                       ds >= 0 ? (float2*)(ws + p.st[ds]) : nullptr};
        return launch(ctx, kUntimed, st, [&] { rn_finish_save_kernel<<<dim3(RN_GROUPS, B, 1), RN_THREADS, 0, st>>>(f, s); });
    };
    auto head = [&](int a) {
        const float* xs[RN_MAX_IN] = {act(a)};
        return rn_launch_head(ctx, st, B, 1, &n, xs, 0, out, ld);
    };
    return rn_walk(ctx, conv, finish, [] { return cudaSuccess; }, head);
}

extern "C" int ssb_smt_resnet18_train_forward_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W,
                                                    const float* d_labels, int n_labels, int64_t label_stride,
                                                    const ssb_resnet_conv convs[20], const float* d_fc_weight,
                                                    const float* d_fc_bias, int fc_in, int n_out, float* d_out,
                                                    void* d_workspace, void* stream) {
    static const char* fn = "ssb_smt_resnet18_train_forward_batch";
    return abi_call(ctx, [&]() -> int {
        SrnPlan p;
        GsRange ins[4 + 3 * RN_CONVS];
        int n_ins = 0;
        const int rc = srn_check(ctx, fn, B, d_spec, H, W, d_labels, n_labels, label_stride, convs, d_fc_weight,
                                 d_fc_bias, fc_in, n_out, d_workspace, &p, ins, &n_ins);
        if (rc != SSB_OK) return rc;
        const GsRange outs[] = {{d_out, (size_t)B * n_out * sizeof(float)}, {d_workspace, (size_t)p.total * sizeof(float)}};
        if (!d_out || misaligned4(d_out) || gs_aliased(outs, 2, ins, n_ins))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad output (NULL, misaligned or overlapping buffers refused)", fn);
        if (B == 0) return SSB_OK;
        const RnNet net{d_spec, convs, d_fc_weight, d_fc_bias, n_out, 0, p.L, {}, nullptr, nullptr};
        return srn_forward(ctx, (cudaStream_t)stream, p, (float*)d_workspace, B, net, true, d_labels,
                           (long long)label_stride, d_out, n_out);
    });
}

// conv dW of layer l (rc rows per chunk; obs: the stem reading the observation's two ears) into the chunk partials,
// then their reduction into dw (row stride Kw); nothing when dw is NULL
static int srn_conv_dw(ssb_ctx* ctx, cudaStream_t st, const RnLayer& l, int rc, bool obs, int B, const float* x,
                       const float* dz, const int* live, const int* count, float* part, float* dw) {
    if (!dw) return SSB_OK;
    SrnConvB c{};
    c.x = x, c.dz = dz, c.out = part, c.live = live, c.count = count;
    c.IC = obs ? 2 : l.ic, c.OC = l.oc, c.H = l.h, c.W = l.w, c.HO = l.ho, c.WO = l.wo, c.stride = l.stride;
    c.pad = l.pad, c.K = c.IC * l.ks * l.ks, c.rc = rc;
    const int tn = 4096 / l.tm;
    const dim3 grid((unsigned)((B + c.rc - 1) / c.rc), (unsigned)((c.K + tn - 1) / tn), (unsigned)((l.oc + l.tm - 1) / l.tm));
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        if (obs && l.tm == 16) srn_dw_kernel<7, true, 16><<<grid, RN_THREADS, 0, st>>>(c);      // SMT stem
        else if (obs) srn_dw_kernel<7, true, 64><<<grid, RN_THREADS, 0, st>>>(c);           // torchvision stem
        else if (l.ks == 7) srn_dw_kernel<7, false, 16><<<grid, RN_THREADS, 0, st>>>(c);    // SMTCNN stem
        else if (l.ks == 3 && l.tm == 16) srn_dw_kernel<3, false, 16><<<grid, RN_THREADS, 0, st>>>(c);
        else if (l.ks == 3 && l.tm == 32) srn_dw_kernel<3, false, 32><<<grid, RN_THREADS, 0, st>>>(c);
        else if (l.ks == 3) srn_dw_kernel<3, false, 64><<<grid, RN_THREADS, 0, st>>>(c);
        else if (l.tm == 32) srn_dw_kernel<1, false, 32><<<grid, RN_THREADS, 0, st>>>(c);
        else srn_dw_kernel<1, false, 64><<<grid, RN_THREADS, 0, st>>>(c);
    }));
    const int Kw = l.ic * l.ks * l.ks;
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        srn_dw_reduce_kernel<<<(l.oc * c.K + 255) / 256, 256, 0, st>>>(part, count, c.rc, l.oc, c.K, Kw, dw);
    }));
    return SSB_OK;
}

// conv dX of layer l (not the stem): out = dX + add
static cudaError_t srn_conv_dx(ssb_ctx* ctx, cudaStream_t st, const RnLayer& l, int B, const float* w,
                               const float* dz, const float* add, const int* count, float* out) {
    SrnConvB c{};
    c.dz = dz, c.w = w, c.add = add, c.out = out, c.count = count;
    c.IC = l.ic, c.OC = l.oc, c.H = l.h, c.W = l.w, c.HO = l.ho, c.WO = l.wo, c.stride = l.stride, c.pad = l.pad;
    const int tm = l.ic <= 16 ? 16 : l.ic <= 32 ? 32 : 64, tn = 4096 / tm;
    const dim3 grid((unsigned)(((long long)B * l.h * l.w + tn - 1) / tn), (unsigned)((l.ic + tm - 1) / tm));
    return launch(ctx, kUntimed, st, [&] {
        if (l.ks == 3 && tm == 16) srn_dx_kernel<3, 16><<<grid, RN_THREADS, 0, st>>>(c);
        else if (l.ks == 3 && tm == 32) srn_dx_kernel<3, 32><<<grid, RN_THREADS, 0, st>>>(c);
        else if (l.ks == 3) srn_dx_kernel<3, 64><<<grid, RN_THREADS, 0, st>>>(c);
        else if (tm == 16) srn_dx_kernel<1, 16><<<grid, RN_THREADS, 0, st>>>(c);
        else if (tm == 32) srn_dx_kernel<1, 32><<<grid, RN_THREADS, 0, st>>>(c);
        else srn_dx_kernel<1, 64><<<grid, RN_THREADS, 0, st>>>(c);
    });
}

// The backward of the blocks, last to first, on the workspace ws of layout p: g[0] holds the gradient of a block's
// output on entry and of its input on exit, x0 is block 0's input.  norm_bwd(i, gin, ds, dsb) launches the norm
// backward of finish i from gin into g[1] (and the downsample conv ds's into g[2]), the identity branch's gradient
// into dsb unless it is NULL.
template <class NormBwd>
static int rn_walk_back(ssb_ctx* ctx, cudaStream_t st, const RnWork& p, float* ws, const float* x0, int B,
                        const ssb_resnet_conv* convs, float* const* d_dweight, NormBwd&& norm_bwd) {
    const RnLayer* L = p.L;
    const int* live = (const int*)(ws + p.live);
    const int* count = live + B;
    float *G = ws + p.g[0], *DZA = ws + p.g[1], *DZD = ws + p.g[2], *DY = ws + p.g[3], *DSB = ws + p.g[4];
    float* part = ws + p.part;
    for (int b = 7; b >= 0; --b) {
        const int c1 = kRnBlocks[b][0], c2 = c1 + 1, cd = kRnBlocks[b][1];
        const float* xin = b == 0 ? x0 : ws + p.y[kRnBlocks[b - 1][0] + 1];
        SSB_CUDA(ctx, norm_bwd(c2, G, cd, cd >= 0 ? nullptr : DSB));
        int r = srn_conv_dw(ctx, st, L[c2], p.rc[c2], false, B, ws + p.y[c1], DZA, live, count, part, d_dweight[c2]);
        if (r) return r;
        SSB_CUDA(ctx, srn_conv_dx(ctx, st, L[c2], B, convs[c2].d_weight, DZA, nullptr, count, DY));
        SSB_CUDA(ctx, norm_bwd(c1, DY, -1, nullptr));
        r = srn_conv_dw(ctx, st, L[c1], p.rc[c1], false, B, xin, DZA, live, count, part, d_dweight[c1]);
        if (r) return r;
        if (cd >= 0) {
            r = srn_conv_dw(ctx, st, L[cd], p.rc[cd], false, B, xin, DZD, live, count, part, d_dweight[cd]);
            if (r) return r;
            SSB_CUDA(ctx, srn_conv_dx(ctx, st, L[cd], B, convs[cd].d_weight, DZD, nullptr, count, DSB));
        }
        SSB_CUDA(ctx, srn_conv_dx(ctx, st, L[c1], B, convs[c1].d_weight, DZA, DSB, count, G));
    }
    return SSB_OK;
}

// The backward of srn_forward from the gradient d_dpred (row stride ld) of its head's n_out columns: the live rows,
// fc, the blocks, the stem (net.x read as the observation when obs, with the label channels' dW from p.NL labels)
// and every norm's dgamma / dbeta.  80 launches, 82 with labels, with every gradient requested.
static int srn_backward(ssb_ctx* ctx, cudaStream_t st, const SrnPlan& p, float* ws, int B, const RnNet& net, bool obs,
                        const float* d_labels, long long label_stride, const float* d_dpred, int ld,
                        float* const* d_dweight, float* const* d_dgamma, float* const* d_dbeta, float* d_dfc_weight,
                        float* d_dfc_bias) {
    const RnLayer* L = p.L;
    const ssb_resnet_conv* convs = net.convs;
    const int n_out = net.n_out;
    int* live = (int*)(ws + p.live);
    const int* count = live + B;
    float *G = ws + p.g[0], *DZA = ws + p.g[1], *DZD = ws + p.g[2];
    float* gpart = ws + p.gpart;
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        srn_live_kernel<<<1, 1024, 0, st>>>(d_dpred, B, n_out, ld, live, live + B);
    }));
    const float* feat = ws + p.y[RN_CONVS - 1];
    const int F = p.feat;
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        srn_fc_dw_kernel<<<dim3((F + 255) / 256, n_out), 256, 0, st>>>(d_dpred, feat, live, count, ld, F,
                                                                        d_dfc_weight, d_dfc_bias);
    }));
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        srn_fc_dx_kernel<<<dim3((F + 255) / 256, B), 256, 0, st>>>(d_dpred, net.fc_w, live, count, n_out, ld, F, G);
    }));
    auto branch = [&](int i, float* dz) {
        return SrnNormBranch{ws + p.z[i], (const float2*)(ws + p.st[i]), convs[i].d_gamma, dz, p.col[i]};
    };
    // GroupNorm backward of finish i (output y[i], gradient gin), with downsample conv ids or an identity residual
    auto norm_bwd = [&](int i, const float* gin, int ids, float* ds) {
        SrnNormBwd nb{};
        nb.gin = gin, nb.y = ws + p.y[i], nb.ds = ds, nb.gpart = gpart, nb.a = branch(i, DZA);
        if (ids >= 0) nb.d = branch(ids, DZD);
        nb.live = live, nb.count = count, nb.C = L[i].oc, nb.P = L[i].ho * L[i].wo, nb.CT = p.CT;
        return launch(ctx, kUntimed, st, [&] {
            srn_norm_bwd_kernel<<<dim3(RN_GROUPS, B), RN_THREADS, 0, st>>>(nb);
        });
    };
    int rc = rn_walk_back(ctx, st, p, ws, ws + p.y[0], B, convs, d_dweight, norm_bwd);
    if (rc != SSB_OK) return rc;
    SSB_CUDA(ctx, norm_bwd(0, G, -1, nullptr));
    rc = srn_conv_dw(ctx, st, L[0], p.rc[0], obs, B, net.x, DZA, live, count, ws + p.part, d_dweight[0]);
    if (rc != SSB_OK) return rc;
    if (p.NL && d_dweight[0]) {
        float* taps = ws + p.taps;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            srn_tap_kernel<<<dim3(L[0].oc, B), 256, 0, st>>>(DZA, count, L[0].oc, L[0].h, L[0].w, taps);
        }));
        const int n = L[0].oc * p.NL * 49;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            srn_label_dw_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_labels, label_stride, taps, live, count,
                                                                 L[0].oc, p.NL, L[0].ic * 49, d_dweight[0]);
        }));
    }
    SrnGnOut o{};
    for (int i = 0; i < RN_CONVS; ++i)
        o.dgamma[i] = d_dgamma[i], o.dbeta[i] = d_dbeta[i], o.C[i] = L[i].oc, o.col[i] = p.col[i];
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        srn_gn_reduce_kernel<<<dim3(1, RN_CONVS), 256, 0, st>>>(gpart, count, p.CT, o);
    }));
    return SSB_OK;
}

extern "C" int ssb_smt_resnet18_train_backward_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W,
                                                     const float* d_labels, int n_labels, int64_t label_stride,
                                                     const ssb_resnet_conv convs[20], const float* d_fc_weight,
                                                     int fc_in, int n_out, const float* d_dpred, void* d_workspace,
                                                     float* const d_dweight[20], float* const d_dgamma[20],
                                                     float* const d_dbeta[20], float* d_dfc_weight, float* d_dfc_bias,
                                                     void* stream) {
    static const char* fn = "ssb_smt_resnet18_train_backward_batch";
    return abi_call(ctx, [&]() -> int {
        SrnPlan p;
        GsRange ins[7 + 6 * RN_CONVS];
        int n_ins = 0;
        int rc = srn_check(ctx, fn, B, d_spec, H, W, d_labels, n_labels, label_stride, convs, d_fc_weight, nullptr,
                           fc_in, n_out, d_workspace, &p, ins, &n_ins);
        if (rc != SSB_OK) return rc;
        rc = rn_check_grads(ctx, fn, p, B, fc_in, n_out, n_out, d_dpred, d_workspace, d_dweight, d_dgamma, d_dbeta,
                            d_dfc_weight, d_dfc_bias, ins, &n_ins);
        if (rc != SSB_OK || B == 0) return rc;
        const RnNet net{d_spec, convs, d_fc_weight, nullptr, n_out, 0, p.L, {}, nullptr, nullptr};
        return srn_backward(ctx, (cudaStream_t)stream, p, (float*)d_workspace, B, net, true, d_labels,
                            (long long)label_stride, d_dpred, n_out, d_dweight, d_dgamma, d_dbeta, d_dfc_weight,
                            d_dfc_bias);
    });
}

// ssb_resnet18_train_*: in training mode the batch mean and variance per channel as st (mean, var, then the FP64
// mean); the maxpool output and its window indices after the layers; the statistics' chunk sums after the forward's
// partial sums; the backward's own buffers are the norm chunk sums and coefficients and the pooled features.
struct BrnPlan : RnWork {
    int hp, wp, rcn[RN_CONVS], chunks[RN_CONVS];
    long long pool, arg, pa, sums, nsum[2], coef[2], pooled;
};

static int brn_plan(ssb_ctx* ctx, const char* fn, int B, int H, int W, int n_out, BrnPlan* p) {
    if (B < 0 || H < 1 || W < 1 || n_out < 1)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d H=%d W=%d n_out=%d)", fn, B, H, W, n_out);
    if (B > SRN_MAX_ENVS) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %d rows > %d", fn, B, SRN_MAX_ENVS);
    if (H > RN_MAX_HW || W > RN_MAX_HW) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %dx%d input > %dx%d", fn, H, W, RN_MAX_HW, RN_MAX_HW);
    p->feat = rn_geometry(false, 2, H, W, p->L);
    p->hp = p->L[1].h, p->wp = p->L[1].w;
    long long pa, pd, sums = 0;
    long long off = rn_work_layers(p, B, [](const RnLayer& l) { return 4LL * l.oc; }, &pa, &pd, 0);
    for (int i = 0; i < RN_CONVS; ++i) {
        p->rcn[i] = std::max(1, BRN_CHUNK / (p->L[i].ho * p->L[i].wo));
        p->chunks[i] = (B + p->rcn[i] - 1) / p->rcn[i];
        sums = std::max(sums, 4LL * p->chunks[i] * p->L[i].oc);    // a double2 per (chunk, channel)
    }
    const long long np = (long long)B * p->L[0].oc * p->hp * p->wp;
    p->pool = off, off += srn_round(np);
    p->arg = off, off += srn_round((np + 3) / 4);                // one byte per pooled value
    p->pa = off, p->sums = off + srn_round(std::max(pa, pd));    // the downsample convs share the partial sums
    const long long fwd_end = p->sums + srn_round(sums);
    off = rn_work_grads(p, B, off, 2);
    for (int k = 0; k < 2; ++k) p->nsum[k] = off, off += srn_round(sums);
    for (int k = 0; k < 2; ++k) p->coef[k] = off, off += 8LL * 512;     // a double4 per channel, C <= 512
    p->pooled = off, off += srn_round((long long)B * p->feat);
    p->total = std::max(off, fwd_end);
    return SSB_OK;
}

extern "C" int64_t ssb_resnet18_train_workspace_bytes(int B, int H, int W, int n_out) {
    BrnPlan p;
    if (brn_plan(nullptr, "", B, H, W, n_out, &p) != SSB_OK) return -1;
    return p.total * (int64_t)sizeof(float);
}

// the arguments both train entries share; then the caller's read-only buffers (the running statistics only in eval
// mode: training writes them)
static int brn_check(ssb_ctx* ctx, const char* fn, int B, const float* d_spec, int H, int W,
                     const ssb_resnet_conv* convs, const float* d_fc_weight, const float* d_fc_bias, int fc_in,
                     int n_out, int bn_training, const void* d_workspace, BrnPlan* p, GsRange* ins, int* n_ins) {
    int rc = brn_plan(ctx, fn, B, H, W, n_out, p);
    if (rc != SSB_OK) return rc;
    rc = rn_train_check(ctx, fn, false, !bn_training, "spectrogram", d_spec, (size_t)B * H * W * 2 * sizeof(float), "",
                        convs, d_fc_weight, d_fc_bias, fc_in, n_out, d_workspace, p->L, [&]() -> int {
        if (bn_training != 0 && bn_training != 1) SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bn_training=%d, not 0 or 1", fn, bn_training);
        return SSB_OK;
    }, ins, n_ins);
    if (rc != SSB_OK) return rc;
    if (fc_in != p->feat) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: fc takes %d features, expected %d", fn, fc_in, p->feat);
    return SSB_OK;
}

extern "C" int ssb_resnet18_train_forward_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W,
                                                const ssb_resnet_conv convs[20], const float* d_fc_weight,
                                                const float* d_fc_bias, int fc_in, int n_out, int bn_training,
                                                float momentum, int64_t* const d_num_batches_tracked[20], float* d_out,
                                                void* d_workspace, void* stream) {
    static const char* fn = "ssb_resnet18_train_forward_batch";
    return abi_call(ctx, [&]() -> int {
        BrnPlan p;
        GsRange ins[4 + 5 * RN_CONVS];
        int n_ins = 0;
        const int rc = brn_check(ctx, fn, B, d_spec, H, W, convs, d_fc_weight, d_fc_bias, fc_in, n_out, bn_training,
                                 d_workspace, &p, ins, &n_ins);
        if (rc != SSB_OK) return rc;
        if (!(momentum >= 0.f && momentum <= 1.f))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: momentum %g outside [0, 1]", fn, (double)momentum);
        int64_t* const* nbt = bn_training ? d_num_batches_tracked : nullptr;
        GsRange outs[2 + 3 * RN_CONVS];
        int n_outs = 0;
        outs[n_outs++] = {d_out, (size_t)B * n_out * sizeof(float)};
        outs[n_outs++] = {d_workspace, (size_t)p.total * sizeof(float)};
        bool bad = !d_out || misaligned4(d_out);
        for (int i = 0; i < RN_CONVS && bn_training; ++i) {
            outs[n_outs++] = {convs[i].d_mean, (size_t)p.L[i].oc * sizeof(float)};
            outs[n_outs++] = {convs[i].d_var, (size_t)p.L[i].oc * sizeof(float)};
            if (nbt) {
                outs[n_outs++] = {nbt[i], nbt[i] ? sizeof(int64_t) : 0};
                bad = bad || ((uintptr_t)nbt[i] & 7u);
            }
        }
        if (bad || gs_aliased(outs, n_outs, ins, n_ins))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad output (NULL, misaligned or overlapping buffers refused)", fn);
        for (int i = 0; i < RN_CONVS && bn_training && B > 0; ++i)
            if ((long long)B * p.L[i].ho * p.L[i].wo == 1)
                SSB_FAIL(ctx, SSB_E_SHAPE, "%s: norm %d has 1 value per channel; training needs more than 1", fn, i);
        if (B == 0) return SSB_OK;
        const cudaStream_t st = (cudaStream_t)stream;
        float* ws = (float*)d_workspace;
        const RnLayer* L = p.L;
        double2* sums = (double2*)(ws + p.sums);
        const RnNet net{d_spec, convs, d_fc_weight, d_fc_bias, n_out, 0, L, {}, ws + p.pa, ws + p.pa};
        auto act = [&](int a) -> const float* { return a < 0 ? d_spec : a == 0 ? ws + p.pool : ws + p.y[a]; };
        // conv i, its sums z[i] and, training, the batch statistics and the running update: 2 or 3 launches
        auto conv = [&](int i, int in, bool ds) -> cudaError_t {
            const float* xs[RN_MAX_IN] = {act(in)};
            cudaError_t e = rn_launch_conv(ctx, st, i, i == 0, B, 1, &net, xs, ds, nullptr, 0);
            const RnLayer& l = L[i];
            const int P = l.ho * l.wo;
            const BrnStats s{net.PA, ws + p.z[i], bn_training ? sums : nullptr, B, l.oc, P, l.S, p.rcn[i]};
            if (e == cudaSuccess)
                e = launch(ctx, kUntimed, st, [&] { brn_stats_kernel<<<dim3(l.oc, p.chunks[i]), RN_THREADS, 0, st>>>(s); });
            if (e != cudaSuccess || !bn_training) return e;
            const BrnUpdate u{sums, ws + p.z[i], ws + p.st[i], ws + p.st[i] + l.oc,
                              (double*)(ws + p.st[i] + 2 * l.oc), (float*)convs[i].d_mean, (float*)convs[i].d_var,
                              nbt ? nbt[i] : nullptr, (long long)B * P, l.oc, P, p.chunks[i], momentum};
            return launch(ctx, kUntimed, st, [&] { brn_update_kernel<<<(l.oc + 255) / 256, 256, 0, st>>>(u); });
        };
        auto norm = [&](int i) {
            const ssb_resnet_conv& c = convs[i];
            return bn_training ? RnNorm{c.d_gamma, c.d_beta, ws + p.st[i], ws + p.st[i] + L[i].oc, c.eps}
                               : RnNorm{c.d_gamma, c.d_beta, c.d_mean, c.d_var, c.eps};
        };
        // rn_forward's finish on z: in eval mode the same arithmetic on the same sums as ssb_resnet18_batch
        auto finish = [&](int i, int res, int ds) {
            RnFinish f{};
            f.in[0] = RnFinishIn{ws + p.z[i], ds >= 0 ? ws + p.z[ds] : nullptr, res >= 0 ? act(res) : nullptr,
                                 ws + p.y[i], norm(i), ds >= 0 ? norm(ds) : RnNorm{}, 1, ds >= 0 ? 1 : 0};
            f.B = B, f.C = L[i].oc, f.P = L[i].ho * L[i].wo, f.relu = 1;
            return launch(ctx, kUntimed, st, [&] { rn_finish_kernel<<<dim3(RN_GROUPS, B, 1), RN_THREADS, 0, st>>>(f); });
        };
        auto tail = [&] { return rn_maxpool(ctx, st, L, B, ws + p.y[0], ws + p.pool, (unsigned char*)(ws + p.arg)); };
        auto head = [&](int a) {
            const float* xs[RN_MAX_IN] = {act(a)};
            return rn_launch_head(ctx, st, B, 1, &net, xs, 1, d_out, n_out);
        };
        return rn_walk(ctx, conv, finish, tail, head);
    });
}

extern "C" int ssb_resnet18_train_backward_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W,
                                                 const ssb_resnet_conv convs[20], const float* d_fc_weight, int fc_in,
                                                 int n_out, int bn_training, const float* d_dpred, void* d_workspace,
                                                 float* const d_dweight[20], float* const d_dgamma[20],
                                                 float* const d_dbeta[20], float* d_dfc_weight, float* d_dfc_bias,
                                                 void* stream) {
    static const char* fn = "ssb_resnet18_train_backward_batch";
    return abi_call(ctx, [&]() -> int {
        BrnPlan p;
        GsRange ins[7 + 8 * RN_CONVS];
        int n_ins = 0;
        int rc = brn_check(ctx, fn, B, d_spec, H, W, convs, d_fc_weight, nullptr, fc_in, n_out, bn_training,
                           d_workspace, &p, ins, &n_ins);
        if (rc != SSB_OK) return rc;
        rc = rn_check_grads(ctx, fn, p, B, fc_in, n_out, n_out, d_dpred, d_workspace, d_dweight, d_dgamma, d_dbeta,
                            d_dfc_weight, d_dfc_bias, ins, &n_ins);
        if (rc != SSB_OK || B == 0) return rc;
        const cudaStream_t st = (cudaStream_t)stream;
        float* ws = (float*)d_workspace;
        const RnLayer* L = p.L;
        int* live = (int*)(ws + p.live);
        const int* count = live + B;
        float *G = ws + p.g[0], *DZA = ws + p.g[1], *DZD = ws + p.g[2], *DY = ws + p.g[3];
        float* pooled = ws + p.pooled;
        const int F = p.feat, P4 = L[RN_CONVS - 1].ho * L[RN_CONVS - 1].wo;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { brn_iota_kernel<<<(B + 256) / 256, 256, 0, st>>>(B, live); }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            brn_pool_kernel<<<B, RN_THREADS, 0, st>>>(ws + p.y[RN_CONVS - 1], F, P4, pooled);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            srn_fc_dw_kernel<<<dim3((F + 255) / 256, n_out), 256, 0, st>>>(d_dpred, pooled, live, count, n_out, F,
                                                                            d_dfc_weight, d_dfc_bias);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            brn_fc_dx_kernel<<<dim3((F + 255) / 256, B), 256, 0, st>>>(d_dpred, d_fc_weight, n_out, F, P4, G);
        }));
        auto branch = [&](int i, float* dz, int k) {
            BrnBranch q{};
            q.z = ws + p.z[i];
            q.mean = bn_training ? ws + p.st[i] : convs[i].d_mean;
            q.var = bn_training ? ws + p.st[i] + L[i].oc : convs[i].d_var;
            q.dmean = bn_training ? (const double*)(ws + p.st[i] + 2 * L[i].oc) : nullptr;
            q.gamma = convs[i].d_gamma, q.sums = (double2*)(ws + p.nsum[k]), q.coef = (double4*)(ws + p.coef[k]);
            q.dz = dz, q.dgamma = d_dgamma[i], q.dbeta = d_dbeta[i], q.eps = convs[i].eps;
            return q;
        };
        // BatchNorm backward of finish i (output y[i], gradient gin), with downsample conv ids or an identity residual:
        // 3 launches
        auto norm_bwd = [&](int i, const float* gin, int ids, float* ds) -> cudaError_t {
            BrnNormBwd nb{};
            nb.gin = gin, nb.y = ws + p.y[i], nb.ds = ds, nb.a = branch(i, DZA, 0);
            if (ids >= 0) nb.d = branch(ids, DZD, 1);
            nb.B = B, nb.C = L[i].oc, nb.P = L[i].ho * L[i].wo, nb.rc = p.rcn[i], nb.chunks = p.chunks[i];
            nb.training = bn_training;
            const dim3 grid(L[i].oc, p.chunks[i]);
            cudaError_t e = launch(ctx, kUntimed, st, [&] { brn_norm_sum_kernel<<<grid, RN_THREADS, 0, st>>>(nb); });
            if (e == cudaSuccess)
                e = launch(ctx, kUntimed, st, [&] {
                    brn_norm_total_kernel<<<dim3((L[i].oc + 255) / 256, ids >= 0 ? 2 : 1), 256, 0, st>>>(nb);
                });
            if (e == cudaSuccess)
                e = launch(ctx, kUntimed, st, [&] { brn_norm_bwd_kernel<<<grid, RN_THREADS, 0, st>>>(nb); });
            return e;
        };
        rc = rn_walk_back(ctx, st, p, ws, ws + p.pool, B, convs, d_dweight, norm_bwd);
        if (rc != SSB_OK) return rc;
        const long long n0 = (long long)B * L[0].oc * L[0].ho * L[0].wo;
        const int blocks = (int)std::min<long long>((n0 + 255) / 256, (long long)ctx->sm_count * 16);
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            brn_maxpool_bwd_kernel<<<blocks, 256, 0, st>>>(G, (const unsigned char*)(ws + p.arg), B * L[0].oc, L[0].ho,
                                                           L[0].wo, p.hp, p.wp, DY);
        }));
        SSB_CUDA(ctx, norm_bwd(0, DY, -1, nullptr));
        return srn_conv_dw(ctx, st, L[0], p.rc[0], true, B, d_spec, DZA, live, count, ws + p.part, d_dweight[0]);
    });
}

#define CNN_MAX_HW 1024     // ssb_smt_cnn_batch: H, W limit of an observation
#define CNN_MAX_RESIZED (64 * CNN_MAX_HW)   // the largest side ResizeCenterCropper's resize gives within that limit

// The pointers and scalars of input k of an ssb_smt_cnn_* call.
static int cnn_check_args(ssb_ctx* ctx, const char* fn, int k, const ssb_smt_cnn_input& in) {
    if (!in.d_obs || misaligned4(in.d_obs) || in.C < 1 || (in.scale != 0 && in.scale != 1) || !in.d_fc_weight ||
        misaligned4(in.d_fc_weight) || misaligned4(in.d_fc_bias) || in.n_out < 1)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad input %d (C=%d scale=%d n_out=%d)", fn, k, in.C, in.scale, in.n_out);
    return SSB_OK;
}

// The shape of input k: the observation, the crop, and fc_in against the network's geometry, which L[k] receives.
static int cnn_check_shape(ssb_ctx* ctx, const char* fn, int k, const ssb_smt_cnn_input& in, RnLayer (*L)[RN_CONVS]) {
    if (in.H < 1 || in.H > CNN_MAX_HW || in.W < 1 || in.W > CNN_MAX_HW)
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: input %d is %dx%d, outside 1..%d", fn, k, in.H, in.W, CNN_MAX_HW);
    if (in.resized_h < CNN_CROP || in.resized_h > CNN_MAX_RESIZED || in.resized_w < CNN_CROP ||
        in.resized_w > CNN_MAX_RESIZED || in.crop_y < 0 || in.crop_x < 0 || in.crop_y > in.resized_h - CNN_CROP ||
        in.crop_x > in.resized_w - CNN_CROP)
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: input %d: a %dx%d crop at (%d, %d) does not lie inside the %dx%d resize", fn, k,
                 CNN_CROP, CNN_CROP, in.crop_y, in.crop_x, in.resized_h, in.resized_w);
    const int feat = rn_geometry(true, in.C, CNN_CROP, CNN_CROP, L[k]);
    if (in.fc_in != feat)
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: input %d: fc takes %d features; the %dx%d crop yields %d", fn, k, in.fc_in,
                 CNN_CROP, CNN_CROP, feat);
    return SSB_OK;
}

// cnn_prep_kernel's arguments for n_inputs inputs writing their images at img[k]
static CnnPrep cnn_prep(int B, int n_inputs, const ssb_smt_cnn_input* inputs, float* const* img) {
    CnnPrep prep{};
    prep.B = B;
    for (int k = 0; k < n_inputs; ++k) {
        const ssb_smt_cnn_input& in = inputs[k];
        prep.in[k] = CnnPrepIn{in.d_obs, img[k], in.scale ? 1.0f / 255.0f : 1.0f, in.C, in.H, in.W, in.resized_h,
                               in.resized_w, in.crop_y, in.crop_x};
    }
    return prep;
}

extern "C" int ssb_smt_cnn_batch(ssb_ctx* ctx, int B, int n_inputs, const ssb_smt_cnn_input* inputs, float* d_out,
                                 void* stream) {
    return abi_call(ctx, [&]() -> int {
        const char* fn = "ssb_smt_cnn_batch";
        if (B < 0 || n_inputs < 1 || n_inputs > RN_MAX_IN || !inputs || !d_out || misaligned4(d_out))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d n_inputs=%d)", fn, B, n_inputs);
        for (int k = 0; k < n_inputs; ++k) {
            int rc = cnn_check_args(ctx, fn, k, inputs[k]);
            if (rc) return rc;
            char what[32];
            snprintf(what, sizeof what, "input %d ", k);
            rc = rn_check_convs(ctx, fn, true, inputs[k].convs, what);
            if (rc) return rc;
        }
        if (B > RN_MAX_ENVS) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %d envs > %d", fn, B, RN_MAX_ENVS);
        RnLayer L[RN_MAX_IN][RN_CONVS];
        RnNet nets[RN_MAX_IN];
        int ld = 0;
        for (int k = 0; k < n_inputs; ++k) {
            const ssb_smt_cnn_input& in = inputs[k];
            const int rc = cnn_check_shape(ctx, fn, k, in, L);
            if (rc) return rc;
            nets[k] = RnNet{nullptr, in.convs, in.d_fc_weight, in.d_fc_bias, in.n_out, ld, L[k], {}, nullptr, nullptr};
            ld += in.n_out;
        }
        if (B == 0) return SSB_OK;
        // scratch per input: the cropped image, then the network's activations and partial sums
        size_t img[RN_MAX_IN], act[RN_MAX_IN], pa[RN_MAX_IN], per[RN_MAX_IN], total = 0;
        for (int k = 0; k < n_inputs; ++k) {
            img[k] = ((size_t)B * inputs[k].C * CNN_CROP * CNN_CROP + 3) & ~(size_t)3;
            per[k] = img[k] + rn_scratch(L[k], B, &act[k], &pa[k]);
            total += per[k];
        }
        SSB_CUDA(ctx, grow_scratch(ctx->nscratch, ctx->nscratch_elems, (total + 1) / 2));
        float* buf = (float*)ctx->nscratch;
        float* x[RN_MAX_IN] = {};
        for (int k = 0; k < n_inputs; ++k) {
            float* a = buf + img[k];
            nets[k].x = x[k] = buf;
            nets[k].A[0] = a, nets[k].A[1] = a + act[k], nets[k].A[2] = a + 2 * act[k];
            nets[k].PA = a + 3 * act[k], nets[k].PD = nets[k].PA + pa[k];
            buf += per[k];
        }
        const CnnPrep prep = cnn_prep(B, n_inputs, inputs, x);
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            cnn_prep_kernel<<<dim3(CNN_CROP * CNN_CROP / 256, B, n_inputs), 256, 0, st>>>(prep);
        }));
        return rn_forward(ctx, st, true, false, B, n_inputs, nets, nullptr, 0, d_out, ld);
    });
}

// ssb_smt_cnn_train_*: the inputs' 64 x 64 images (the stem's dW reads them), then each network laid out as
// ssb_smt_resnet18_train_* lays out one, without labels and with a dW GEMM over all C stem channels.  Every network's
// total is the end of the whole workspace, so each network's output checks cover all of it.
struct CnnTrainPlan {
    SrnPlan net[RN_MAX_IN];
    long long img[RN_MAX_IN], total;
    int ld;                 // the sum of the n_out: d_out's and d_dout's row stride
};

static int cnn_train_plan(ssb_ctx* ctx, const char* fn, int B, int n_inputs, const ssb_smt_cnn_input* inputs,
                          CnnTrainPlan* p) {
    if (B < 0 || n_inputs < 1 || n_inputs > RN_MAX_IN || !inputs)
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d n_inputs=%d)", fn, B, n_inputs);
    for (int k = 0; k < n_inputs; ++k) {
        const int rc = cnn_check_args(ctx, fn, k, inputs[k]);
        if (rc) return rc;
    }
    if (B > SRN_MAX_ENVS) SSB_FAIL(ctx, SSB_E_SHAPE, "%s: %d rows > %d", fn, B, SRN_MAX_ENVS);
    long long off = 0;
    RnLayer L[RN_MAX_IN][RN_CONVS];
    for (int k = 0; k < n_inputs; ++k) {
        const int rc = cnn_check_shape(ctx, fn, k, inputs[k], L);
        if (rc) return rc;
        std::copy(L[k], L[k] + RN_CONVS, p->net[k].L);
        p->img[k] = off, off += srn_round((long long)B * inputs[k].C * CNN_CROP * CNN_CROP);
    }
    p->ld = 0;
    for (int k = 0; k < n_inputs; ++k) {
        SrnPlan& q = p->net[k];
        q.NL = 0, q.feat = inputs[k].fc_in;
        srn_layout(&q, B, off, inputs[k].C);
        off = q.total;
        p->ld += inputs[k].n_out;
    }
    p->total = off;
    for (int k = 0; k < n_inputs; ++k) p->net[k].total = off;
    return SSB_OK;
}

extern "C" int64_t ssb_smt_cnn_train_workspace_bytes(int B, int n_inputs, const ssb_smt_cnn_input* inputs) {
    CnnTrainPlan p;
    if (cnn_train_plan(nullptr, "", B, n_inputs, inputs, &p) != SSB_OK) return -1;
    return p.total * (int64_t)sizeof(float);
}

// the arguments both train entries share: the plan, then per input rn_train_check; then the read-only buffers
static int cnn_train_check(ssb_ctx* ctx, const char* fn, int B, int n_inputs, const ssb_smt_cnn_input* inputs,
                           const void* d_workspace, CnnTrainPlan* p, GsRange* ins, int* n_ins) {
    int rc = cnn_train_plan(ctx, fn, B, n_inputs, inputs, p);
    for (int k = 0; k < n_inputs && rc == SSB_OK; ++k) {
        const ssb_smt_cnn_input& in = inputs[k];
        char name[32], what[32];
        snprintf(name, sizeof name, "input %d observation", k);
        snprintf(what, sizeof what, "input %d ", k);
        rc = rn_train_check(ctx, fn, true, false, name, in.d_obs, (size_t)B * in.H * in.W * in.C * sizeof(float), what,
                            in.convs, in.d_fc_weight, in.d_fc_bias, in.fc_in, in.n_out, d_workspace, p->net[k].L,
                            [] { return (int)SSB_OK; }, ins, n_ins);
    }
    return rc;
}

// input k's first column in d_out and d_dout
static int cnn_col(const ssb_smt_cnn_input* inputs, int k) {
    int col = 0;
    for (int j = 0; j < k; ++j) col += inputs[j].n_out;
    return col;
}

// input k's network for srn_forward / srn_backward: its image, parameters and output columns
static RnNet cnn_train_net(const CnnTrainPlan& p, const ssb_smt_cnn_input* inputs, int k, float* ws) {
    const ssb_smt_cnn_input& in = inputs[k];
    return RnNet{ws + p.img[k], in.convs, in.d_fc_weight, in.d_fc_bias, in.n_out, cnn_col(inputs, k), p.net[k].L, {},
                 nullptr, nullptr};
}

extern "C" int ssb_smt_cnn_train_forward_batch(ssb_ctx* ctx, int B, int n_inputs, const ssb_smt_cnn_input* inputs,
                                               float* d_out, void* d_workspace, void* stream) {
    static const char* fn = "ssb_smt_cnn_train_forward_batch";
    return abi_call(ctx, [&]() -> int {
        CnnTrainPlan p;
        GsRange ins[RN_MAX_IN * (3 + 3 * RN_CONVS)];
        int n_ins = 0;
        const int rc = cnn_train_check(ctx, fn, B, n_inputs, inputs, d_workspace, &p, ins, &n_ins);
        if (rc != SSB_OK) return rc;
        const GsRange outs[] = {{d_out, (size_t)B * p.ld * sizeof(float)}, {d_workspace, (size_t)p.total * sizeof(float)}};
        if (!d_out || misaligned4(d_out) || gs_aliased(outs, 2, ins, n_ins))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad output (NULL, misaligned or overlapping buffers refused)", fn);
        if (B == 0) return SSB_OK;
        const cudaStream_t st = (cudaStream_t)stream;
        float* ws = (float*)d_workspace;
        float* img[RN_MAX_IN] = {};
        for (int k = 0; k < n_inputs; ++k) img[k] = ws + p.img[k];
        const CnnPrep prep = cnn_prep(B, n_inputs, inputs, img);
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            cnn_prep_kernel<<<dim3(CNN_CROP * CNN_CROP / 256, B, n_inputs), 256, 0, st>>>(prep);
        }));
        for (int k = 0; k < n_inputs; ++k) {
            const int r = srn_forward(ctx, st, p.net[k], ws, B, cnn_train_net(p, inputs, k, ws), false, nullptr, 0,
                                      d_out, p.ld);
            if (r != SSB_OK) return r;
        }
        return SSB_OK;
    });
}

extern "C" int ssb_smt_cnn_train_backward_batch(ssb_ctx* ctx, int B, int n_inputs, const ssb_smt_cnn_input* inputs,
                                                const float* d_dout, void* d_workspace, float* const* d_grads,
                                                void* stream) {
    static const char* fn = "ssb_smt_cnn_train_backward_batch";
    return abi_call(ctx, [&]() -> int {
        CnnTrainPlan p;
        GsRange ins[RN_MAX_IN * (6 + 6 * RN_CONVS)];
        int n_ins = 0;
        int rc = cnn_train_check(ctx, fn, B, n_inputs, inputs, d_workspace, &p, ins, &n_ins);
        if (rc != SSB_OK) return rc;
        if (!d_grads) SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad gradient arguments (NULL gradient table)", fn);
        for (int k = 0; k < n_inputs; ++k) {
            const ssb_smt_cnn_input& in = inputs[k];
            float* const* g = d_grads + CNN_TRAIN_GRADS * k;
            rc = rn_check_grads(ctx, fn, p.net[k], B, in.fc_in, in.n_out, p.ld, d_dout ? d_dout + cnn_col(inputs, k) : nullptr,
                                d_workspace, g, g + RN_CONVS, g + 2 * RN_CONVS, g[3 * RN_CONVS], g[3 * RN_CONVS + 1],
                                ins, &n_ins);
            if (rc != SSB_OK) return rc;
        }
        if (B == 0) return SSB_OK;
        const cudaStream_t st = (cudaStream_t)stream;
        float* ws = (float*)d_workspace;
        for (int k = 0; k < n_inputs; ++k) {
            const RnNet net = cnn_train_net(p, inputs, k, ws);
            float* const* g = d_grads + CNN_TRAIN_GRADS * k;
            rc = srn_backward(ctx, st, p.net[k], ws, B, net, false, nullptr, 0, d_dout + net.col, p.ld, g,
                              g + RN_CONVS, g + 2 * RN_CONVS, g[3 * RN_CONVS], g[3 * RN_CONVS + 1]);
            if (rc != SSB_OK) return rc;
        }
        return SSB_OK;
    });
}

// per-env valid-token counts at the head of the scratch, padded to 256 bytes
static int64_t smt_cnt_bytes(int B) { return ((int64_t)B * (int64_t)sizeof(int) + 255) / 256 * 256; }

extern "C" int64_t ssb_smt_scratch_bytes(int B, int M, const ssb_smt_params* p) {
    if (!p || B < 0 || M < 0 || p->d_model < 1) return -1;
    return smt_cnt_bytes(B) + 5LL * B * (M + 1) * p->d_model * (int64_t)sizeof(float);
}

static bool smt_bad_linear(const ssb_linear& l) {
    return !l.d_weight || !l.d_bias || misaligned4(l.d_weight) || misaligned4(l.d_bias);
}

static bool smt_bad_norm(const ssb_layer_norm& n) {
    return !n.d_gamma || !n.d_beta || misaligned4(n.d_gamma) || misaligned4(n.d_beta) || !(n.eps > 0.f);
}

// The argument checks all three ssb_smt_state_encoder_* entries make, in this order; max_B: the entry's row limit.
static int smt_check(ssb_ctx* ctx, const char* fn, int B, int M, const float* d_x, const float* d_memory,
                     const float* d_masks, const float* d_goal, const ssb_smt_params* p, const void* d_ws,
                     const float* d_out, int max_B) {
    if (B < 0 || M < 0 || !p || !d_x || misaligned4(d_x) || !d_out || misaligned4(d_out) || !d_ws ||
        ((uintptr_t)d_ws & 15u) || misaligned4(d_goal) ||
        (M > 0 && (!d_memory || !d_masks || misaligned4(d_memory) || misaligned4(d_masks))))
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d M=%d)", fn, B, M);
    if (p->d_in < 1 || p->pose_index < -1 || p->n_heads < 1 || p->d_model < 1 || p->d_model % p->n_heads ||
        (p->pretraining != 0 && p->pretraining != 1))
        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad parameters (d_in=%d pose_index=%d d_model=%d n_heads=%d "
                 "pretraining=%d)", fn, p->d_in, p->pose_index, p->d_model, p->n_heads, p->pretraining);
    const ssb_linear* lins[] = {&p->fuse1, &p->fuse2, &p->enc_qkv, &p->enc_out, &p->enc_ff1, &p->enc_ff2,
                                &p->dec_sa_qkv, &p->dec_sa_out, &p->dec_ca_qkv, &p->dec_ca_out, &p->dec_ff1,
                                &p->dec_ff2, &p->pose};
    for (int i = 0; i < 13; ++i)
        if ((i < 12 || p->pose_index >= 0) && smt_bad_linear(*lins[i]))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: NULL or misaligned linear parameter %d", fn, i);
    const ssb_layer_norm* norms[] = {&p->enc_norm1, &p->enc_norm2, &p->enc_norm, &p->dec_norm1, &p->dec_norm2,
                                     &p->dec_norm3, &p->dec_norm};
    for (int i = 0; i < 7; ++i)
        if (smt_bad_norm(*norms[i]))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad LayerNorm %d (eps=%g)", fn, i, (double)norms[i]->eps);
    const int d = p->d_model, hd = d / p->n_heads;
    if (B > max_B || M + 1 > SMT_MAX_TOKENS || d > SMT_MAX_D || hd > SMT_MAX_HD || p->d_in > SMT_MAX_IN ||
        (p->pose_index >= 0 && p->pose_index + 4 > p->d_in))
        SSB_FAIL(ctx, SSB_E_SHAPE, "%s: B=%d M=%d d_model=%d head dim=%d d_in=%d pose_index=%d outside the limits "
                 "(B <= %d, M + 1 <= %d, d_model <= %d, head dim <= %d, d_in <= %d, pose_index + 4 <= d_in)", fn, B,
                 M, d, hd, p->d_in, p->pose_index, max_B, SMT_MAX_TOKENS, SMT_MAX_D, SMT_MAX_HD, SMT_MAX_IN);
    return SSB_OK;
}

// The kernels' view of the inputs and parameters; the activation pointers are the caller's.
static SmtArgs smt_args(int B, int M, const float* d_x, const float* d_memory, const float* d_masks,
                        const float* d_goal, const ssb_smt_params* p, float* d_out) {
    SmtArgs a;
    memset(&a, 0, sizeof(a));
    const int d = p->d_model;
    a.x = d_x, a.memory = d_memory, a.masks = d_masks, a.goal = d_goal, a.out = d_out;
    auto lin = [](const ssb_linear& l, size_t row0, int in) {
        return SmtLin{l.d_weight + row0 * in, l.d_bias + row0};
    };
    auto ln = [](const ssb_layer_norm& n) { return SmtLn{n.d_gamma, n.d_beta, n.eps}; };
    const int F = p->pose_index >= 0 ? p->pose_index + 16 : p->d_in;
    a.pose = p->pose_index >= 0 ? lin(p->pose, 0, 5) : SmtLin{nullptr, nullptr};
    a.fuse1 = lin(p->fuse1, 0, F), a.fuse2 = lin(p->fuse2, 0, d);
    a.enc_qkv = lin(p->enc_qkv, 0, d), a.enc_out = lin(p->enc_out, 0, d);
    a.enc_ff1 = lin(p->enc_ff1, 0, d), a.enc_ff2 = lin(p->enc_ff2, 0, d);
    a.dec_v = lin(p->dec_sa_qkv, 2 * (size_t)d, d), a.dec_sa_out = lin(p->dec_sa_out, 0, d);
    a.dec_q = lin(p->dec_ca_qkv, 0, d), a.dec_kv = lin(p->dec_ca_qkv, d, d), a.dec_ca_out = lin(p->dec_ca_out, 0, d);
    a.dec_ff1 = lin(p->dec_ff1, 0, d), a.dec_ff2 = lin(p->dec_ff2, 0, d);
    a.enc_n1 = ln(p->enc_norm1), a.enc_n2 = ln(p->enc_norm2), a.enc_n = ln(p->enc_norm);
    a.dec_n1 = ln(p->dec_norm1), a.dec_n2 = ln(p->dec_norm2), a.dec_n3 = ln(p->dec_norm3), a.dec_n = ln(p->dec_norm);
    a.B = B, a.M = M, a.T = M + 1, a.d_in = p->d_in, a.pi = p->pose_index, a.F = F, a.d = d, a.H = p->n_heads;
    a.hd = d / p->n_heads;
    a.pretraining = p->pretraining;
    return a;
}

// The six launches of the forward, on whatever buffers a points at.
static int smt_forward(ssb_ctx* ctx, const SmtArgs& a, cudaStream_t st) {
    const int d = a.d, hd = a.hd, T = a.T, B = a.B;
    const unsigned tiles = (unsigned)((T + SMT_RT - 1) / SMT_RT);
    const int Fp = (a.F + 3) & ~3, Tp = (T + 3) & ~3;
    const size_t sm_fuse = (size_t)(SMT_RT * Fp + SMT_RT * d + SMT_WS + SMT_RT + 8) * 4;
    const size_t sm_lin = (size_t)(SMT_RT * d + SMT_WS) * 4;
    const size_t sm_attn = (size_t)(SMT_RT * hd + SMT_KT_KEYS * (hd + 1) + SMT_RT * Tp) * 4;
    const size_t sm_tail = (size_t)(3 * SMT_RT * d + SMT_WS) * 4;
    const size_t sm_dec = (size_t)(4 * SMT_DEC_ENVS * d + 8 * Tp) * 4;
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { smt_fuse_kernel<<<dim3(tiles, B), SMT_THREADS, sm_fuse, st>>>(a); }));
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        smt_linear_kernel<<<dim3(tiles, (3 * d + 127) / 128, B), SMT_THREADS, sm_lin, st>>>(
            a.cnt, a.h0, d, T, d, a.enc_qkv, 3 * d, a.qkv, 3 * d);
    }));
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        smt_attn_kernel<<<dim3(tiles, a.H, B), SMT_THREADS, sm_attn, st>>>(a);
    }));
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { smt_enc_tail_kernel<<<dim3(tiles, B), SMT_THREADS, sm_tail, st>>>(a); }));
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        smt_linear_kernel<<<dim3(tiles, (2 * d + 127) / 128, B), SMT_THREADS, sm_lin, st>>>(
            a.cnt, a.enc, d, T, d, a.dec_kv, 2 * d, a.kv, 2 * d);
    }));
    SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
        smt_decoder_kernel<<<(B + SMT_DEC_ENVS - 1) / SMT_DEC_ENVS, SMT_THREADS, sm_dec, st>>>(a);
    }));
    return SSB_OK;
}

extern "C" int ssb_smt_state_encoder_batch(ssb_ctx* ctx, int B, int M, const float* d_x, const float* d_memory,
                                           const float* d_masks, const float* d_goal, const ssb_smt_params* p,
                                           void* d_scratch, float* d_out, void* stream) {
    return abi_call(ctx, [&]() -> int {
        const char* fn = "ssb_smt_state_encoder_batch";
        const int rc = smt_check(ctx, fn, B, M, d_x, d_memory, d_masks, d_goal, p, d_scratch, d_out, SMT_MAX_ENVS);
        if (rc != SSB_OK) return rc;
        if (B == 0) return SSB_OK;
        SmtArgs a = smt_args(B, M, d_x, d_memory, d_masks, d_goal, p, d_out);
        const size_t rows = (size_t)B * a.T * a.d;
        a.cnt = (int*)d_scratch;
        a.h0 = (float*)((char*)d_scratch + smt_cnt_bytes(B));
        a.qkv = a.h0 + rows;
        a.att = a.qkv + 3 * rows;
        a.enc = a.att, a.kv = a.qkv;
        return smt_forward(ctx, a, (cudaStream_t)stream);
    });
}

// ssb_smt_state_encoder_train_*: the workspace, laid out from base (sizes only when base is 0), into g (g->f: the
// forward's buffers, with nothing overwritten in place).  Returns its bytes.  Every region is 256-byte aligned.
static int64_t smt_train_plan(int B, int M, const ssb_smt_params* p, uintptr_t base, SmtBwdArgs* g) {
    SmtArgs& a = g->f;
    const int64_t T = M + 1, d = p->d_model, BT = (int64_t)B * T, H = p->n_heads;
    const int64_t F = p->pose_index >= 0 ? p->pose_index + 16 : p->d_in, Fp = (F + 3) & ~3;
    int64_t off = 0;
    auto take = [&](int64_t floats) {
        float* r = (float*)(base + off);
        off += (floats * 4 + 255) / 256 * 256;
        return r;
    };
    a.cnt = (int*)take(B), a.slot = (int*)take(BT);
    a.h0 = take(BT * d), a.qkv = take(BT * 3 * d), a.att = take(BT * d), a.enc = take(BT * d), a.kv = take(BT * 2 * d);
    a.xin = take(BT * Fp), a.hid = take(BT * d), a.u = take(BT * 2 * d), a.ffh = take(BT * d), a.st = take(BT * 6);
    float** tok[] = {&g->dE, &g->datt, &g->du1, &g->du2, &g->dfp, &g->a1, &g->xn, &g->dn2, &g->x2, &g->da1, &g->x1,
                     &g->dh0b, &g->dh0, &g->dhp};
    for (float** t : tok) *t = take(BT * d);
    g->dkv = take(BT * 2 * d), g->dqkv = take(BT * 3 * d);
    g->dpe = take(BT * 16), g->pf = take(BT * 8), g->posec = take(BT * 4), g->ast = take(BT * H * 3);
    for (int i = 0; i < SMT_DEC_BUFS; ++i) g->dec[i] = take((int64_t)B * d);
    const int64_t wt_n[SMT_N_WT] = {F, d, 3 * d, d, d, d, 2 * d, d, d, d, d, d, d};   // rows of W^T, each d wide
    for (int i = 0; i < SMT_N_WT; ++i) g->wt[i] = take(wt_n[i] * d);
    g->zeros = take(std::max(3 * d, Fp));
    g->S = std::max(1, std::min(B, SMT_DW_SPLITS));
    // (x, ldx, dy, ldy, K, N, per_env, diag) of each sum
    float* const* D = g->dec;
    const struct { const float* x; int64_t ldx; const float* dy; int64_t ldy, K, N; int per_env, diag; } js[SMT_JOBS] = {
        {a.xin, Fp, g->dhp, d, F, d, 0, 0},         {a.hid, d, g->dh0, d, d, d, 0, 0},
        {a.h0, d, g->dqkv, 3 * d, d, 3 * d, 0, 0},  {a.att, d, g->du1, d, d, d, 0, 0},
        {g->a1, d, g->dfp, d, d, d, 0, 0},          {a.ffh, d, g->du2, d, d, d, 0, 0},
        {a.enc, d, g->dkv, 2 * d, d, 2 * d, 0, 0},  {g->pf, 8, g->dpe, 16, 5, p->pose_index >= 0 ? 16 : 0, 0, 0},
        {D[SD_T0], d, D[SD_DV], d, d, d, 1, 0},     {D[SD_V], d, D[SD_DU1], d, d, d, 1, 0},
        {D[SD_N1], d, D[SD_DQ], d, d, d, 1, 0},     {D[SD_CC], d, D[SD_DU2], d, d, d, 1, 0},
        {D[SD_N2], d, D[SD_DFFP], d, d, d, 1, 0},   {D[SD_FF], d, D[SD_DU3], d, d, d, 1, 0},
        {g->x1, d, g->da1, d, d, d, 0, 1},          {g->x2, d, g->dn2, d, d, d, 0, 1},
        {g->xn, d, g->dE, d, d, d, 0, 1},           {D[SD_XH1], d, D[SD_DY1], d, d, d, 1, 1},
        {D[SD_XH2], d, D[SD_DY2], d, d, d, 1, 1},   {D[SD_XH3], d, D[SD_DY3], d, d, d, 1, 1},
        {D[SD_XHN], d, D[SD_DYN], d, d, d, 1, 1}};
    for (int i = 0; i < SMT_JOBS; ++i) {
        SmtDwJob& j = g->jobs[i];
        j.x = js[i].x, j.dy = js[i].dy, j.ldx = (int)js[i].ldx, j.ldy = (int)js[i].ldy, j.K = (int)js[i].K;
        j.N = (int)js[i].N, j.per_env = js[i].per_env, j.diag = js[i].diag;
        j.part = j.N ? take((int64_t)g->S * (j.diag ? 2 * j.N : j.N * (j.K + 1))) : nullptr;
        j.outw = j.outb = nullptr;
    }
    return off;
}

extern "C" int64_t ssb_smt_train_workspace_bytes(int B, int M, const ssb_smt_params* p) {
    if (!p || B < 0 || B > SMT_MAX_TRAIN_ENVS || M < 0 || M + 1 > SMT_MAX_TOKENS || p->d_model < 1 ||
        p->n_heads < 1 || p->d_in < 1 || p->pose_index < -1 || p->d_in > SMT_MAX_IN)
        return -1;
    SmtBwdArgs g;
    memset(&g, 0, sizeof(g));
    return smt_train_plan(B, M, p, 0, &g);
}

extern "C" int ssb_smt_state_encoder_train_forward_batch(ssb_ctx* ctx, int B, int M, const float* d_x,
                                                         const float* d_memory, const float* d_masks,
                                                         const float* d_goal, const ssb_smt_params* p,
                                                         void* d_workspace, float* d_out, void* stream) {
    return abi_call(ctx, [&]() -> int {
        const char* fn = "ssb_smt_state_encoder_train_forward_batch";
        const int rc = smt_check(ctx, fn, B, M, d_x, d_memory, d_masks, d_goal, p, d_workspace, d_out,
                                 SMT_MAX_TRAIN_ENVS);
        if (rc != SSB_OK) return rc;
        if (B == 0) return SSB_OK;
        SmtBwdArgs g;
        memset(&g, 0, sizeof(g));
        g.f = smt_args(B, M, d_x, d_memory, d_masks, d_goal, p, d_out);
        smt_train_plan(B, M, p, (uintptr_t)d_workspace, &g);
        return smt_forward(ctx, g.f, (cudaStream_t)stream);
    });
}

extern "C" int ssb_smt_state_encoder_train_backward_batch(ssb_ctx* ctx, int B, int M, const float* d_x,
                                                          const float* d_memory, const float* d_masks,
                                                          const float* d_goal, const ssb_smt_params* p,
                                                          const float* d_dout, int ld_dout, void* d_workspace,
                                                          float* const* d_grads, float* d_dx, float* d_dgoal,
                                                          void* stream) {
    return abi_call(ctx, [&]() -> int {
        const char* fn = "ssb_smt_state_encoder_train_backward_batch";
        const int rc = smt_check(ctx, fn, B, M, d_x, d_memory, d_masks, d_goal, p, d_workspace, d_dout,
                                 SMT_MAX_TRAIN_ENVS);
        if (rc != SSB_OK) return rc;
        if (!d_grads || ld_dout < p->d_model || misaligned4(d_dx) || misaligned4(d_dgoal) || (d_dgoal && !d_goal))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad gradient arguments (ld_dout=%d)", fn, ld_dout);
        const int o = p->pose_index >= 0 ? 2 : 0, ng = 38 + o;
        for (int i = 0; i < ng; ++i)
            if (misaligned4(d_grads[i]))
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: misaligned gradient %d", fn, i);
        if (B == 0) return SSB_OK;
        SmtBwdArgs g;
        memset(&g, 0, sizeof(g));
        g.f = smt_args(B, M, d_x, d_memory, d_masks, d_goal, p, nullptr);
        smt_train_plan(B, M, p, (uintptr_t)d_workspace, &g);
        const SmtArgs& a = g.f;
        const int d = a.d, T = a.T;
        g.dout = d_dout, g.ld_dout = ld_dout, g.dx = d_dx, g.dgoal = d_dgoal;
        // gradient table: ssb_smt_params order, pose_encoder's two first when it has them
        float* const* G = d_grads + o;
        const int out_idx[SMT_JOBS] = {0, 2, 4, 6, 8, 10, 22, -2, 18, 20, 22, 24, 26, 28, 12, 14, 16, 30, 32, 34, 36};
        const int64_t row_off[SMT_JOBS] = {0, 0, 0, 0, 0, 0, d, 0, 2 * d, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (int i = 0; i < SMT_JOBS; ++i) {
            SmtDwJob& j = g.jobs[i];
            float* w = i == SJ_POSE && !o ? nullptr : G[out_idx[i]];
            float* b = i == SJ_POSE && !o ? nullptr : G[out_idx[i] + 1];
            j.outw = w ? w + row_off[i] * (j.diag ? 0 : j.K) : nullptr;
            j.outb = b ? b + row_off[i] : nullptr;
            if (!j.outw && !j.outb) j.part = nullptr;     // not asked for: its launches' CTAs exit
        }
        g.zero_w = G[18], g.zero_b = G[19];
        const cudaStream_t st = (cudaStream_t)stream;
        // transposed weights of the dX GEMMs (SW_* order)
        SmtTArgs t;
        memset(&t, 0, sizeof(t));
        const SmtLin lw[SMT_N_WT] = {a.fuse1, a.fuse2, a.enc_qkv, a.enc_out, a.enc_ff1, a.enc_ff2, a.dec_kv, a.dec_v,
                                     a.dec_sa_out, a.dec_q, a.dec_ca_out, a.dec_ff1, a.dec_ff2};
        const int tn[SMT_N_WT] = {d, d, 3 * d, d, d, d, 2 * d, d, d, d, d, d, d};
        int tmax = 0;
        for (int i = 0; i < SMT_N_WT; ++i) {
            const int K = i == SW_FUSE1 ? a.F : d;
            t.job[i] = SmtTJob{lw[i].w, (float*)g.wt[i], tn[i], K};
            tmax = std::max(tmax, ((tn[i] + 31) / 32) * ((K + 31) / 32));
        }
        t.zeros = (float*)g.zeros, t.nz = std::max(3 * d, (a.F + 3) & ~3);
        const unsigned tiles = (unsigned)((T + SMT_RT - 1) / SMT_RT);
        const int Fp = (a.F + 3) & ~3, Tp = (T + 3) & ~3;
        const size_t sm_dec = (size_t)(14 * SMT_DEC_ENVS * d + 16 * Tp) * 4;
        const size_t sm_tail = (size_t)(3 * SMT_RT * d + SMT_WS) * 4;
        const size_t sm_attn = (size_t)16 * Tp * 4;
        const size_t sm_fuse = (size_t)(2 * SMT_RT * d + SMT_RT * Fp + SMT_WS) * 4;
        int dw_tiles = 0;
        size_t red = 2 * (size_t)d * d;
        if (a.pi >= 0) red = std::max(red, (size_t)B * (a.d_in - a.pi));
        for (const SmtDwJob& j : g.jobs) {
            if (!j.N) continue;
            const int k1 = (j.K + 1 + SMT_DW_TILE - 1) / SMT_DW_TILE, n1 = (j.N + SMT_DW_TILE - 1) / SMT_DW_TILE;
            dw_tiles = std::max(dw_tiles, j.diag ? (j.N + SMT_THREADS - 1) / SMT_THREADS : k1 * n1);
            red = std::max(red, j.diag ? 2 * (size_t)j.N : (size_t)j.N * (j.K + 1));
        }
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            smt_transpose_kernel<<<dim3(tmax, SMT_N_WT), SMT_THREADS, 0, st>>>(t);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            smt_dec_bwd_kernel<<<(B + SMT_DEC_ENVS - 1) / SMT_DEC_ENVS, SMT_THREADS, sm_dec, st>>>(g);
        }));
        const size_t sm_lin2 = (size_t)(SMT_RT * 2 * d + SMT_WS) * 4, sm_lin3 = (size_t)(SMT_RT * 3 * d + SMT_WS) * 4;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            smt_linear_kernel<<<dim3(tiles, (d + 127) / 128, B), SMT_THREADS, sm_lin2, st>>>(
                a.cnt, g.dkv, 2 * d, T, 2 * d, SmtLin{g.wt[SW_KV], g.zeros}, d, g.dE, d);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            smt_enc_tail_bwd_kernel<<<dim3(tiles, B), SMT_THREADS, sm_tail, st>>>(g);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            smt_attn_bwd_kernel<false><<<dim3(tiles, a.H, B), SMT_THREADS, sm_attn, st>>>(g);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            smt_attn_bwd_kernel<true><<<dim3(tiles, a.H, B), SMT_THREADS, sm_attn, st>>>(g);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            smt_linear_kernel<<<dim3(tiles, (d + 127) / 128, B), SMT_THREADS, sm_lin3, st>>>(
                a.cnt, g.dqkv, 3 * d, T, 3 * d, SmtLin{g.wt[SW_QKV], g.zeros}, d, g.dh0b, d);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            smt_fuse_bwd_kernel<<<dim3(tiles, B), SMT_THREADS, sm_fuse, st>>>(g);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            smt_dw_kernel<<<dim3(dw_tiles, g.S, SMT_JOBS), SMT_THREADS, 0, st>>>(g);
        }));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            smt_reduce_kernel<<<dim3((unsigned)((red + SMT_THREADS - 1) / SMT_THREADS), SMT_JOBS + 2), SMT_THREADS,
                                0, st>>>(g);
        }));
        return SSB_OK;
    });
}

extern "C" int ssb_pcm16_decode(ssb_ctx* ctx, const int16_t* d_in, int64_t n, float* d_out, void* stream) {
    return abi_call(ctx, [&]() -> int {
        if (n == 0) return SSB_OK;
        if (n < 0 || !d_in || !d_out) SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_pcm16_decode: bad arguments");
        int blocks = (int)((n + 255) / 256);
        if (blocks > ctx->sm_count * 16) blocks = ctx->sm_count * 16;
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { pcm16_decode_kernel<<<blocks, 256, 0, st>>>(d_in, (long long)n, d_out); }));
        return SSB_OK;
    });
}

extern "C" int ssb_pcm16_encode(ssb_ctx* ctx, const float* d_in, int64_t n, int mode, int16_t* d_out, void* stream) {
    return abi_call(ctx, [&]() -> int {
        if (n == 0) return SSB_OK;
        if (n < 0 || !d_in || !d_out || (mode != 0 && mode != 1)) SSB_FAIL(ctx, SSB_E_INVALID_ARG, "ssb_pcm16_encode: bad arguments");
        int blocks = (int)((n + 255) / 256);
        if (blocks > ctx->sm_count * 16) blocks = ctx->sm_count * 16;
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { pcm16_encode_kernel<<<blocks, 256, 0, st>>>(d_in, (long long)n, mode, d_out); }));
        return SSB_OK;
    });
}

// ---------------------------------------------------------------------------
// AV-WaN's maps on the device: replay of Mapper.reset / Mapper.update and the three egocentric crops
// (include/ssb200.h, ssb_map_update_batch / ssb_map_observe_batch)
// ---------------------------------------------------------------------------
constexpr int MAPK_THREADS = 256;
constexpr int MAPK_TILE = 32;             // geometric-map output tile (rows x cells) staged in shared memory

struct MapGeo {
    int n, s, S, a, E, enc, acoustic, m;  // m = n / s, the acoustic map's side
    long long pitch;                      // SSB_MAP_PITCH(n)
};

// (row, col) of the unrotated n x n map that np.rot90(map, k)[r][c] reads
__host__ __device__ __forceinline__ void map_unrot(int k, int n, int r, int c, int& row, int& col) {
    if (k == 0) { row = r; col = c; }
    else if (k == 1) { row = c; col = n - 1 - r; }
    else if (k == 2) { row = n - 1 - r; col = n - 1 - c; }
    else { row = n - 1 - c; col = r; }
}

// transform_coordinates(x, y, 90 k, n, n) of mapper.py: where cell (x, y) lands in np.rot90(map, k)
__host__ __device__ __forceinline__ void map_rot_xy(int k, int n, int x, int y, int& rx, int& ry) {
    if (k == 0) { rx = x; ry = y; }
    else if (k == 1) { rx = y; ry = n - 1 - x; }
    else if (k == 2) { rx = n - 1 - x; ry = n - 1 - y; }
    else { rx = n - 1 - y; ry = x; }
}

// quarter turns of the mapper's view: rotate_map(map, -self._rotation) with -_rotation = orientation - 270
__host__ __device__ __forceinline__ int map_turns(int orientation) { return ((orientation + 90) % 360) / 90; }

// One CTA per slot touched: ranges[blockIdx.x] = (slot, first record, records, -); records of a slot in order.
// kDeviceIntensity: an update's acoustic value is intensity[r.reserved] (ssb_map_update_device_intensity_batch), the
// Python float a worker's Intensity sensor returns, so half is its float64 product with 0.5; otherwise the record's
// own intensity and half fields (ssb_map_update_batch; `intensity` is unused).
template <bool kDeviceIntensity>
__global__ void __launch_bounds__(MAPK_THREADS) map_update_kernel(MapGeo g, const int4* __restrict__ ranges,
                                                                  const ssb_map_record* __restrict__ rec,
                                                                  const uint8_t* __restrict__ ego,
                                                                  uint8_t* __restrict__ gmap, double* __restrict__ amap,
                                                                  const float* __restrict__ intensity) {
    const int4 rg = ranges[blockIdx.x];
    uint8_t* gm = gmap + (long long)rg.x * g.pitch;
    double* am = g.acoustic ? amap + (long long)rg.x * g.m * g.m : nullptr;
    for (int i = 0; i < rg.z; ++i) {
        const ssb_map_record r = rec[rg.y + i];
        if (r.kind == SSB_MAP_RESET) {
            uint4* p = reinterpret_cast<uint4*>(gm);       // the pitch is a multiple of 16 bytes
            for (long long j = threadIdx.x; j < g.pitch / 16; j += blockDim.x) p[j] = make_uint4(0u, 0u, 0u, 0u);
            if (am)
                for (int j = threadIdx.x; j < g.m * g.m; j += blockDim.x) am[j] = 0.0;
        } else {
            const int k = map_turns(r.orientation);
            int rx, ry;
            map_rot_xy(k, g.n, r.x, r.y, rx, ry);
            const int top = ry - g.E, left = rx - g.E / 2;
            const uint8_t* eb = ego + r.ego_offset;
            // top < 0 only for E = 1 at ry = 0, where the reference's window slice is empty and nothing is written
            for (int j = threadIdx.x; top >= 0 && j < g.E * g.E; j += blockDim.x) {
                // cell j's two bits (channel 0 first, MSB-first packing) share one byte: 2 j is even
                const unsigned two = (eb[j >> 2] >> (6 - 2 * (j & 3))) & 3u;
                if (two) {
                    const int er = j / g.E, ec = j - er * g.E;
                    int row, col;
                    map_unrot(k, g.n, top + er, left + ec, row, col);
                    gm[(long long)row * g.n + col] |= (uint8_t)(((two >> 1) & 1u) | ((two & 1u) << 1));
                }
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                // Mapper.update's loop visits the agent's own node unless it stands within s - 1 cells of the view's
                // far edges (its range() bounds truncate); a visited obstacle there is cleared
                if (rx <= g.n + 1 - g.s && ry <= g.n + 1 - g.s) gm[(long long)r.y * g.n + r.x] &= (uint8_t)~1u;
                if (am) {
                    double value = r.intensity, half = r.half;
                    if constexpr (kDeviceIntensity) {
                        value = (double)intensity[r.reserved];
                        half = __dmul_rn(0.5, value);
                    }
                    double* c = am + (long long)(r.y / g.s) * g.m + r.x / g.s;
                    if (g.enc == SSB_MAP_INTENSITY || *c == 0.0) *c = value;
                    else *c = __dadd_rn(half, __dmul_rn(0.5, *c));
                }
            }
        }
        __syncthreads();
    }
}

// Grid (n_gm_blocks + 1 or n_gm_blocks, B): blocks below n_gm_blocks write one 32 x 32-cell tile of gm; the last
// block of an env writes am and action_map.  The tile is read in the order that is contiguous in the unrotated map
// (output columns for an even number of quarter turns, output rows for an odd one) and written row by row.
__global__ void __launch_bounds__(MAPK_THREADS) map_observe_kernel(MapGeo g, const int4* __restrict__ poses,
                                                                   const int* __restrict__ tables, int L, int tiles_x,
                                                                   int n_gm_blocks, const uint8_t* __restrict__ gmap,
                                                                   const double* __restrict__ amap, float* d_gm,
                                                                   long long gm_stride, float* d_am, long long am_stride,
                                                                   float* d_action, long long action_stride) {
    __shared__ uint8_t tile[MAPK_TILE][MAPK_TILE + 1];
    const int b = blockIdx.y;
    const int4 p = poses[b];                   // (slot, x, y, orientation)
    const int k = map_turns(p.w);
    int rx, ry;
    map_rot_xy(k, g.n, p.y, p.z, rx, ry);
    if ((int)blockIdx.x < n_gm_blocks) {
        const int ti = blockIdx.x / tiles_x, tj = blockIdx.x - ti * tiles_x;
        const int i0 = ti * MAPK_TILE, j0 = tj * MAPK_TILE;
        const int r0 = ry - g.S / 2 + i0, c0 = rx - g.S / 2 + j0;
        const uint8_t* gm = gmap + (long long)p.x * g.pitch;
        for (int e = threadIdx.x; e < MAPK_TILE * MAPK_TILE; e += blockDim.x) {
            const int fast = e % MAPK_TILE, slow = e / MAPK_TILE;
            const int di = (k & 1) ? fast : slow, dj = (k & 1) ? slow : fast;
            const int r = r0 + di, c = c0 + dj;
            uint8_t v = 0;
            if (r >= 0 && r < g.n && c >= 0 && c < g.n) {
                int row, col;
                map_unrot(k, g.n, r, c, row, col);
                v = gm[(long long)row * g.n + col];
            }
            tile[di][dj] = v;
        }
        __syncthreads();
        float* out = d_gm + (long long)b * gm_stride;
        for (int e = threadIdx.x; e < MAPK_TILE * MAPK_TILE * 2; e += blockDim.x) {
            const int di = e / (2 * MAPK_TILE), f = e % (2 * MAPK_TILE), dj = f >> 1, ch = f & 1;
            const int i = i0 + di, j = j0 + dj;
            if (i < g.S && j < g.S) out[((long long)i * g.S + j) * 2 + ch] = (float)((tile[di][dj] >> ch) & 1);
        }
        return;
    }
    if (d_am) {
        constexpr int C = SSB_MAP_AM_CROP;
        int ax, ay;
        map_rot_xy(k, g.m, p.y / g.s, p.z / g.s, ax, ay);
        const double* am = amap + (long long)p.x * g.m * g.m;
        float* out = d_am + (long long)b * am_stride;
        for (int e = threadIdx.x; e < C * C; e += blockDim.x) {
            const int r = ay - C / 2 + e / C, c = ax - C / 2 + e % C;
            double v = 0.0;
            if (r >= 0 && r < g.m && c >= 0 && c < g.m) {
                int row, col;
                map_unrot(k, g.m, r, c, row, col);
                v = am[(long long)row * g.m + col];
            }
            out[e] = __double2float_rn(v);
        }
    }
    if (d_action) {
        const int* xs = tables + 2 * k * L;
        const int* ys = xs + L;
        const int gy = ry / g.s - g.a / 2, gx = rx / g.s - g.a / 2;
        const uint8_t* gm = gmap + (long long)p.x * g.pitch;
        float* out = d_action + (long long)b * action_stride;
        for (int e = threadIdx.x; e < g.a * g.a; e += blockDim.x) {
            int row, col;
            map_unrot(k, g.n, ys[gy + e / g.a], xs[gx + e % g.a], row, col);
            out[e] = (gm[(long long)row * g.n + col] & 1u) ? 0.f : 1.f;
        }
    }
}

static bool map_geometry(const ssb_map_geometry* g, MapGeo* out) {
    if (!g) return false;
    const int n = g->internal_size;
    if (n < 1 || n > SSB_MAP_MAX_INTERNAL || g->stride < 1 || g->stride > n || g->map_size < 2 ||
        g->map_size > SSB_MAP_MAX_INTERNAL || (g->map_size & 1) || g->action_size < 1 ||
        g->action_size > SSB_MAP_MAX_EGO || !(g->action_size & 1) || g->ego_size < 1 || g->ego_size > n ||
        g->ego_size > SSB_MAP_MAX_EGO || (g->encoding != SSB_MAP_INTENSITY && g->encoding != SSB_MAP_AVERAGE_INTENSITY) ||
        (g->acoustic != 0 && g->acoustic != 1) || g->n_slots < 1 || g->n_slots > SSB_MAP_MAX_SLOTS)
        return false;
    *out = MapGeo{n, g->stride, g->map_size, g->action_size, g->ego_size, g->encoding, g->acoustic, n / g->stride,
                  (long long)SSB_MAP_PITCH(n)};
    return true;
}

static bool map_orientation_ok(int o) { return o >= 0 && o < 360 && o % 90 == 0; }

// Host staging of a map entry's inputs (ctx->mstage[which]): waits for the kernel that last read the buffers, grows
// them to `bytes`, returns the pinned host buffer and its device copy.
static int map_stage(ssb_ctx* ctx, int which, size_t bytes, void** h, void** d) {
    ssb_ctx::MapStage& m = ctx->mstage[which];
    if (!m.done) SSB_CUDA(ctx, cudaEventCreateWithFlags(&m.done, cudaEventDisableTiming));
    SSB_CUDA(ctx, cudaEventSynchronize(m.done));
    if (bytes > m.cap) {
        if (m.h) cudaFreeHost(m.h);
        if (m.d) cudaFree(m.d);
        m.h = m.d = nullptr;
        m.cap = 0;
        const size_t cap = std::max(bytes, (size_t)64 * 1024);
        SSB_CUDA(ctx, cudaMallocHost(&m.h, cap));
        SSB_CUDA(ctx, cudaMalloc(&m.d, cap));
        m.cap = cap;
    }
    *h = m.h;
    *d = m.d;
    return SSB_OK;
}

static size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

// Both update entries: the host checks, the staging and the one launch.  kDeviceIntensity: update records of an
// acoustic geometry index d_intensity (n_intensity floats) with their reserved field.
template <bool kDeviceIntensity>
static int map_update_batch(ssb_ctx* ctx, const char* fn, const ssb_map_geometry* geo, uint8_t* d_gmap,
                            double* d_amap, int n_records, const ssb_map_record* h_records, const uint8_t* h_ego,
                            int64_t ego_bytes, const float* d_intensity, int64_t n_intensity, void* stream) {
    return abi_call(ctx, [&]() -> int {
        MapGeo g;
        if (!map_geometry(geo, &g))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad geometry", fn);
        if (n_records < 0 || (n_records > 0 && !h_records) || ego_bytes < 0 || (ego_bytes > 0 && !h_ego) || !d_gmap ||
            ((uintptr_t)d_gmap & 15u) || (g.acoustic && (!d_amap || ((uintptr_t)d_amap & 7u))) || n_intensity < 0)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (n_records=%d ego_bytes=%lld n_intensity=%lld)", fn,
                     n_records, (long long)ego_bytes, (long long)n_intensity);
        const int64_t ego_rec = ((int64_t)g.E * g.E * 2 + 7) / 8;
        for (int i = 0; i < n_records; ++i) {
            const ssb_map_record& r = h_records[i];
            if (r.slot < 0 || r.slot >= geo->n_slots || (r.kind != SSB_MAP_RESET && r.kind != SSB_MAP_UPDATE))
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: record %d: bad slot %d or kind %d", fn, i, r.slot, r.kind);
            if (r.kind == SSB_MAP_RESET) continue;
            if (!map_orientation_ok(r.orientation) || r.ego_offset < 0 || r.ego_offset > ego_bytes - ego_rec)
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: record %d: bad orientation %d or ego offset %lld", fn, i,
                         r.orientation, (long long)r.ego_offset);
            if (kDeviceIntensity && g.acoustic &&
                (!d_intensity || ((uintptr_t)d_intensity & 3u) || r.reserved < 0 || r.reserved >= n_intensity))
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: record %d: intensity index %d outside [0, %lld) or a NULL or "
                         "misaligned d_intensity", fn, i, r.reserved, (long long)n_intensity);
            if (r.x < 0 || r.x >= g.n || r.y < 0 || r.y >= g.n)
                SSB_FAIL(ctx, SSB_E_SHAPE, "%s: record %d: pose (%d, %d) outside the %d x %d map", fn, i, r.x, r.y,
                         g.n, g.n);
            int rx, ry;
            map_rot_xy(map_turns(r.orientation), g.n, r.x, r.y, rx, ry);
            // with E = 1 at ry = 0 the reference's rows [-1, 0) are an empty slice its one-row ego map broadcasts
            // into: it writes nothing and completes the update
            if ((ry - g.E < 0 && g.E > 1) || rx - g.E / 2 < 0 || rx - g.E / 2 + g.E > g.n)
                SSB_FAIL(ctx, SSB_E_SHAPE, "%s: record %d: the %d x %d ego window at (%d, %d) of the rotated view "
                         "leaves the %d x %d map", fn, i, g.E, g.E, rx, ry, g.n, g.n);
            // at stride 1 Mapper.update's loop runs one cell past new_top and new_right, so it reads row N when ry =
            // N - 1 and column N when the window ends at column N - 1 or N, and raises IndexError there
            if (g.s == 1 && (ry == g.n - 1 || rx - g.E / 2 + g.E >= g.n - 1))
                SSB_FAIL(ctx, SSB_E_SHAPE, "%s: record %d: at stride 1 the reference's loop reads past the %d x %d map "
                         "for the agent at (%d, %d) of the rotated view", fn, i, g.n, g.n, rx, ry);
            if (g.acoustic && (r.x / g.s >= g.m || r.y / g.s >= g.m))
                SSB_FAIL(ctx, SSB_E_SHAPE, "%s: record %d: acoustic cell (%d, %d) outside the %d x %d map", fn, i,
                         r.x / g.s, r.y / g.s, g.m, g.m);
        }
        if (n_records == 0) return SSB_OK;
        std::vector<int> order(n_records);
        for (int i = 0; i < n_records; ++i) order[i] = i;
        std::stable_sort(order.begin(), order.end(),
                         [&](int a, int b) { return h_records[a].slot < h_records[b].slot; });
        int n_groups = 0;
        for (int i = 0; i < n_records; ++i)
            n_groups += i == 0 || h_records[order[i]].slot != h_records[order[i - 1]].slot;
        const size_t off_rec = align16((size_t)n_groups * sizeof(int4));
        const size_t off_ego = align16(off_rec + (size_t)n_records * sizeof(ssb_map_record));
        void *h, *d;
        if (int rc = map_stage(ctx, 0, off_ego + (size_t)ego_bytes, &h, &d)) return rc;
        int4* hr = (int4*)h;
        ssb_map_record* hrec = (ssb_map_record*)((char*)h + off_rec);
        for (int i = 0, gi = -1; i < n_records; ++i) {
            const ssb_map_record& r = h_records[order[i]];
            if (i == 0 || r.slot != h_records[order[i - 1]].slot) hr[++gi] = make_int4(r.slot, i, 0, 0);
            hr[gi].z += 1;
            hrec[i] = r;
        }
        if (ego_bytes) memcpy((char*)h + off_ego, h_ego, (size_t)ego_bytes);
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, cudaMemcpyAsync(d, h, off_ego + (size_t)ego_bytes, cudaMemcpyHostToDevice, st));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            map_update_kernel<kDeviceIntensity><<<n_groups, MAPK_THREADS, 0, st>>>(
                g, (const int4*)d, (const ssb_map_record*)((char*)d + off_rec), (const uint8_t*)d + off_ego, d_gmap,
                d_amap, d_intensity);
        }));
        SSB_CUDA(ctx, cudaEventRecord(ctx->mstage[0].done, st));
        return SSB_OK;
    });
}

extern "C" int ssb_map_update_batch(ssb_ctx* ctx, const ssb_map_geometry* geo, uint8_t* d_gmap, double* d_amap,
                                    int n_records, const ssb_map_record* h_records, const uint8_t* h_ego,
                                    int64_t ego_bytes, void* stream) {
    return map_update_batch<false>(ctx, "ssb_map_update_batch", geo, d_gmap, d_amap, n_records, h_records, h_ego,
                                   ego_bytes, nullptr, 0, stream);
}

extern "C" int ssb_map_update_device_intensity_batch(ssb_ctx* ctx, const ssb_map_geometry* geo, uint8_t* d_gmap,
                                                     double* d_amap, int n_records, const ssb_map_record* h_records,
                                                     const uint8_t* h_ego, int64_t ego_bytes, const float* d_intensity,
                                                     int64_t n_intensity, void* stream) {
    return map_update_batch<true>(ctx, "ssb_map_update_device_intensity_batch", geo, d_gmap, d_amap, n_records,
                                  h_records, h_ego, ego_bytes, d_intensity, n_intensity, stream);
}

extern "C" int ssb_map_observe_batch(ssb_ctx* ctx, const ssb_map_geometry* geo, const uint8_t* d_gmap,
                                     const double* d_amap, int B, const int32_t* h_poses, const int32_t* h_tables,
                                     int L, float* d_gm, int64_t gm_stride, float* d_am, int64_t am_stride,
                                     float* d_action, int64_t action_stride, void* stream) {
    static const char* fn = "ssb_map_observe_batch";
    return abi_call(ctx, [&]() -> int {
        MapGeo g;
        if (!map_geometry(geo, &g))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad geometry", fn);
        const bool need_g = d_gm || d_action;
        if (B < 0 || B > SSB_MAP_MAX_SLOTS || (B > 0 && !h_poses) ||
            (need_g && (!d_gmap || ((uintptr_t)d_gmap & 15u))) ||
            (d_am && (!g.acoustic || !d_amap || ((uintptr_t)d_amap & 7u))) ||
            (d_gm && (misaligned4(d_gm) || gm_stride < (int64_t)g.S * g.S * 2)) ||
            (d_am && (misaligned4(d_am) || am_stride < SSB_MAP_AM_CROP * SSB_MAP_AM_CROP)) ||
            (d_action && (misaligned4(d_action) || action_stride < (int64_t)g.a * g.a || L < 1 || !h_tables)))
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (B=%d L=%d gm_stride=%lld am_stride=%lld "
                     "action_stride=%lld)", fn, B, L, (long long)gm_stride, (long long)am_stride,
                     (long long)action_stride);
        if (d_action)
            for (int i = 0; i < 8 * L; ++i)
                if (h_tables[i] < 0 || h_tables[i] >= g.n)
                    SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: navigable table entry %d is %d, outside [0, %d)", fn, i,
                             h_tables[i], g.n);
        for (int b = 0; b < B; ++b) {
            const int32_t* p = h_poses + 4 * b;
            if (p[0] < 0 || p[0] >= geo->n_slots || !map_orientation_ok(p[3]))
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: env %d: bad slot %d or orientation %d", fn, b, p[0], p[3]);
            if (p[1] < 0 || p[1] >= g.n || p[2] < 0 || p[2] >= g.n)
                SSB_FAIL(ctx, SSB_E_SHAPE, "%s: env %d: pose (%d, %d) outside the %d x %d map", fn, b, p[1], p[2],
                         g.n, g.n);
            if (d_am && (p[1] / g.s >= g.m || p[2] / g.s >= g.m))
                SSB_FAIL(ctx, SSB_E_SHAPE, "%s: env %d: acoustic cell (%d, %d) outside the %d x %d map", fn, b,
                         p[1] / g.s, p[2] / g.s, g.m, g.m);
            if (d_action) {
                int rx, ry;
                map_rot_xy(map_turns(p[3]), g.n, p[1], p[2], rx, ry);
                const int gx = rx / g.s, gy = ry / g.s;
                if (gx - g.a / 2 < 0 || gy - g.a / 2 < 0 || gx + g.a / 2 + 1 > L || gy + g.a / 2 + 1 > L)
                    SSB_FAIL(ctx, SSB_E_SHAPE, "%s: env %d: the %d x %d occupancy window at grid cell (%d, %d) "
                             "leaves the %d x %d grid", fn, b, g.a, g.a, gx, gy, L, L);
            }
        }
        const int tiles_x = (g.S + MAPK_TILE - 1) / MAPK_TILE;
        const int n_gm_blocks = d_gm ? tiles_x * tiles_x : 0;
        const int blocks_x = n_gm_blocks + ((d_am || d_action) ? 1 : 0);
        if (B == 0 || blocks_x == 0) return SSB_OK;
        const size_t off_tab = align16((size_t)B * sizeof(int4));
        const size_t tab_bytes = d_action ? (size_t)8 * L * sizeof(int32_t) : 0;
        void *h, *d;
        if (int rc = map_stage(ctx, 1, off_tab + tab_bytes, &h, &d)) return rc;
        memcpy(h, h_poses, (size_t)B * sizeof(int4));
        if (tab_bytes) memcpy((char*)h + off_tab, h_tables, tab_bytes);
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, cudaMemcpyAsync(d, h, off_tab + tab_bytes, cudaMemcpyHostToDevice, st));
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] {
            map_observe_kernel<<<dim3(blocks_x, B), MAPK_THREADS, 0, st>>>(
                g, (const int4*)d, (const int*)((char*)d + off_tab), L, tiles_x, n_gm_blocks, d_gmap, d_amap, d_gm,
                (long long)gm_stride, d_am, (long long)am_stride, d_action, (long long)action_stride);
        }));
        SSB_CUDA(ctx, cudaEventRecord(ctx->mstage[1].done, st));
        return SSB_OK;
    });
}

// ---------------------------------------------------------------------------
// Remote env workers' visual frames (soundspaces_b200.frames): one launch gathers every visual sensor's rows of a step
// from its device frame bank into float32 rows (uint8 converted exactly, float32 copied bit for bit), reading the rows
// uploaded this step from the staging buffer and writing them into their bank rows as well.  blockIdx.z is the
// sensor; blockIdx.y < N gathers destination row y, blockIdx.y >= N stores staged row y - N into its bank row; the
// x blocks stride over the row in 16-byte units (vec) or in elements.
#define FG_THREADS 256
#define FG_MAX_BLOCKS_X 16

struct FgSensor {
    char* bank;
    const char* stage;
    float* dst;
    long long row_elems, dst_stride;
    int n_fill, u8, vec;
};

struct FgParams {
    FgSensor s[SSB_FRAME_MAX_SENSORS];
    int N;
    int index[SSB_FRAME_MAX_SENSORS][SSB_FRAME_MAX_N];   // >= 0: bank row, < 0: staged row -1 - index
    int fill[SSB_FRAME_MAX_SENSORS][SSB_FRAME_MAX_N];    // bank row of staged row j
};

__device__ __forceinline__ float4 fg_u8x4(unsigned w) {
    return make_float4((float)(w & 0xffu), (float)((w >> 8) & 0xffu), (float)((w >> 16) & 0xffu), (float)(w >> 24));
}

__global__ void __launch_bounds__(FG_THREADS) frame_gather_kernel(const __grid_constant__ FgParams p) {
    const FgSensor& s = p.s[blockIdx.z];
    const int r = blockIdx.y;
    const long long row_bytes = s.row_elems << (s.u8 ? 0 : 2);
    const long long t0 = (long long)blockIdx.x * FG_THREADS + threadIdx.x;
    const long long step = (long long)gridDim.x * FG_THREADS;
    if (r >= p.N) {
        const int j = r - p.N;
        if (j >= s.n_fill) return;
        const char* src = s.stage + j * row_bytes;
        char* dst = s.bank + (long long)p.fill[blockIdx.z][j] * row_bytes;
        if (s.vec) {
            for (long long i = t0; i < (row_bytes >> 4); i += step)
                reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
        } else if (s.u8) {
            for (long long i = t0; i < row_bytes; i += step) dst[i] = src[i];
        } else {
            for (long long i = t0; i < s.row_elems; i += step)
                reinterpret_cast<unsigned*>(dst)[i] = reinterpret_cast<const unsigned*>(src)[i];
        }
        return;
    }
    const int ix = p.index[blockIdx.z][r];
    const char* src = ix >= 0 ? s.bank + (long long)ix * row_bytes : s.stage + (long long)(-1 - ix) * row_bytes;
    float* dst = s.dst + (long long)r * s.dst_stride;
    if (s.u8) {
        if (s.vec) {
            for (long long i = t0; i < (s.row_elems >> 4); i += step) {
                const uint4 v = __ldg(reinterpret_cast<const uint4*>(src) + i);
                float4* o = reinterpret_cast<float4*>(dst) + 4 * i;
                o[0] = fg_u8x4(v.x);
                o[1] = fg_u8x4(v.y);
                o[2] = fg_u8x4(v.z);
                o[3] = fg_u8x4(v.w);
            }
        } else {
            const unsigned char* b = reinterpret_cast<const unsigned char*>(src);
            for (long long i = t0; i < s.row_elems; i += step) dst[i] = (float)b[i];
        }
    } else if (s.vec) {                                   // float32 as is: the bits move, NaN payloads included
        for (long long i = t0; i < (row_bytes >> 4); i += step)
            reinterpret_cast<uint4*>(dst)[i] = __ldg(reinterpret_cast<const uint4*>(src) + i);
    } else {
        for (long long i = t0; i < s.row_elems; i += step)
            reinterpret_cast<unsigned*>(dst)[i] = reinterpret_cast<const unsigned*>(src)[i];
    }
}

namespace {
struct FgRegion { uintptr_t lo, hi; bool written; };
}

extern "C" int ssb_frame_gather_batch(ssb_ctx* ctx, int n_sensors, const ssb_frame_sensor* sensors, int N,
                                      void* stream) {
    static const char* fn = "ssb_frame_gather_batch";
    return abi_call(ctx, [&]() -> int {
        if (n_sensors < 1 || n_sensors > SSB_FRAME_MAX_SENSORS || !sensors || N < 0)
            SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: bad arguments (n_sensors=%d N=%d)", fn, n_sensors, N);
        if (N > SSB_FRAME_MAX_N)
            SSB_FAIL(ctx, SSB_E_SHAPE, "%s: N=%d, the kernel is built for N <= %d", fn, N, SSB_FRAME_MAX_N);
        FgParams p;
        memset(&p, 0, sizeof(p));
        p.N = N;
        FgRegion reg[3 * SSB_FRAME_MAX_SENSORS];
        int n_reg = 0;
        long long max_units = 0;
        for (int q = 0; q < n_sensors; ++q) {
            const ssb_frame_sensor& s = sensors[q];
            if (s.dtype != SSB_FRAME_U8 && s.dtype != SSB_FRAME_F32)
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: sensor %d: unsupported dtype %d (SSB_FRAME_U8 or SSB_FRAME_F32)",
                         fn, q, s.dtype);
            const bool u8 = s.dtype == SSB_FRAME_U8;
            if (s.row_elems < 1 || s.bank_rows < 1 || s.dst_stride < s.row_elems || s.n_fill < 0 || s.n_fill > N)
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: sensor %d: bad shape (row_elems=%lld bank_rows=%lld "
                         "dst_stride=%lld n_fill=%d N=%d)", fn, q, (long long)s.row_elems, (long long)s.bank_rows,
                         (long long)s.dst_stride, s.n_fill, N);
            const long long esize = u8 ? 1 : 4;
            if ((double)s.bank_rows * (double)s.row_elems * esize >= (double)(1ll << 46) ||
                (double)(N + 1) * (double)s.dst_stride * 4 >= (double)(1ll << 46))
                SSB_FAIL(ctx, SSB_E_SHAPE, "%s: sensor %d: a bank or destination of 2^46 bytes or more", fn, q);
            if (!s.d_bank || (N > 0 && (!s.d_dst || !s.h_index)) || (s.n_fill > 0 && (!s.d_stage || !s.h_fill)))
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: sensor %d: a NULL pointer the call needs", fn, q);
            if (misaligned4(s.d_dst) || (!u8 && (misaligned4(s.d_bank) || misaligned4(s.d_stage))))
                SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: sensor %d: a float32 buffer not aligned to 4 bytes", fn, q);
            const long long row_bytes = s.row_elems * esize;
            for (int j = 0; j < s.n_fill; ++j) {
                const int32_t f = s.h_fill[j];
                if (f < 0 || f >= s.bank_rows)
                    SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: sensor %d: fill row %d outside [0, %lld)", fn, q, f,
                             (long long)s.bank_rows);
                for (int k = 0; k < j; ++k)
                    if (s.h_fill[k] == f)
                        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: sensor %d: bank row %d is filled twice", fn, q, f);
                p.fill[q][j] = f;
            }
            for (int i = 0; i < N; ++i) {
                const int32_t x = s.h_index[i];
                if (x < -s.n_fill || x >= s.bank_rows)
                    SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: sensor %d: index %d of row %d outside [%d, %lld)", fn, q, x,
                             i, -s.n_fill, (long long)s.bank_rows);
                for (int j = 0; x >= 0 && j < s.n_fill; ++j)
                    if (s.h_fill[j] == x)
                        SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: sensor %d: row %d reads bank row %d, which this call "
                                 "fills (read the staged row instead)", fn, q, i, x);
                p.index[q][i] = x;
            }
            reg[n_reg++] = FgRegion{(uintptr_t)s.d_bank, (uintptr_t)s.d_bank + (uintptr_t)(s.bank_rows * row_bytes),
                                    s.n_fill > 0};
            if (s.n_fill > 0)
                reg[n_reg++] = FgRegion{(uintptr_t)s.d_stage,
                                        (uintptr_t)s.d_stage + (uintptr_t)(s.n_fill * row_bytes), false};
            if (N > 0)
                reg[n_reg++] = FgRegion{(uintptr_t)s.d_dst,
                                        (uintptr_t)(s.d_dst + (N - 1) * s.dst_stride + s.row_elems), true};
            const bool vec = (row_bytes & 15) == 0 && ((uintptr_t)s.d_bank & 15) == 0 &&
                             ((uintptr_t)s.d_stage & 15) == 0 && ((uintptr_t)s.d_dst & 15) == 0 &&
                             (s.dst_stride & 3) == 0;
            p.s[q] = FgSensor{(char*)s.d_bank, (const char*)s.d_stage, s.d_dst, (long long)s.row_elems,
                              (long long)s.dst_stride, s.n_fill, u8 ? 1 : 0, vec ? 1 : 0};
            max_units = std::max(max_units, vec ? row_bytes >> 4 : (long long)s.row_elems);
        }
        for (int a = 0; a < n_reg; ++a)
            for (int b = 0; b < a; ++b)
                if ((reg[a].written || reg[b].written) && reg[a].lo < reg[b].hi && reg[b].lo < reg[a].hi)
                    SSB_FAIL(ctx, SSB_E_INVALID_ARG, "%s: overlapping buffers (a destination or a bank this call "
                             "fills shares bytes with another buffer)", fn);
        if (N == 0) return SSB_OK;
        int max_fill = 0;
        for (int q = 0; q < n_sensors; ++q) max_fill = std::max(max_fill, sensors[q].n_fill);
        const int bx = (int)std::min<long long>(FG_MAX_BLOCKS_X, (max_units + FG_THREADS - 1) / FG_THREADS);
        const dim3 grid(bx, N + max_fill, n_sensors);
        const cudaStream_t st = (cudaStream_t)stream;
        SSB_CUDA(ctx, launch(ctx, kUntimed, st, [&] { frame_gather_kernel<<<grid, FG_THREADS, 0, st>>>(p); }));
        return SSB_OK;
    });
}
