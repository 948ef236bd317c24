// Single-block convolution: ONE 65536-point circular convolution per env, computed by a cluster of 4 CTAs whose
// shared memory holds the env's whole spectrum -- forward FFT of the RIR, pointwise product with the (cached)
// source spectrum and inverse FFT in one kernel, nothing but the waveform leaves the chip.
//
// Replaces, for every request whose RIR is short enough (taps <= 65536 - sr + 1; config 2: 16384 taps at 44.1 kHz,
// config 3: 48000 taps at 16 kHz, head and valid mode alike), the three-kernel partitioned pipeline
// (fwd_rir -> mac_ifft_cluster at N = 4096, fwd_rir -> mac_bins -> mac_ifft at N >= 8192) and its HBM/L2-visible
// intermediates: H (33 MB per 128-env step at config 2), and Y where the sums do not stay on chip, against 21.5 MB of
// algorithmic traffic per step.
//
// Reference semantics (soundspaces/simulator.py:629-647, continuous_simulator.py:428-456; include/ssb200.h):
//     out[m] = sum_k h[k] * x_ext[offset + m - k],   m < out_samples.
// Overlap-save with ONE block of M = 65536: the source segment xs[j] = x_ext[offset - D + j] (j < M) with the shift
// D = M - sr; the circular convolution c = h (*) xs is alias-free at indices >= taps - 1, and out[m] = c[m + D].
//
// Decomposition (DIF radix-16 first stage, 65536 = 16 x 4096): spectrum bin 16 k1 + r belongs to sub-problem r;
//   forward:  a_r[n1] = w_M^(n1 r) * sum_q h[n1 + 4096 q] w16^(q r),  HX_r = FFT4096(a_r)
//   product:  Z_r = HX_r * SX_r                                         (SX_r: source, same layout, cached per clip)
//   inverse:  e_r = IFFT4096(Z_r),  c[n1 + 4096 q] = (1/M) sum_r w16^(-q r) w_M^(-n1 r) e_r[n1].
// CTA c of the cluster owns r = c + 4 m (m = 0..3: one 256-thread group each, running the register-resident
// radix-16 transforms of fft16.cuh on its own exchange buffer with its own named barrier).  With q = q1 + 4 q2 the
// 16-point stages factor into  [radix-4 over q2 / across CTAs] x [radix-4 over q1 / within the CTA]:
//   * forward: every CTA reads the RIR itself (only q2 = 0 is non-zero for taps <= 16384), so NO data crosses CTAs;
//   * inverse: each CTA reduces its four e_r to v_c[q1][n1] in place in shared memory, and the last radix-4 over c
//     reads the three peer CTAs' v through distributed shared memory (96 KB per CTA) -- the only exchange.
// tests/block64_model.py is the numpy model of exactly this data flow (checked against the oracle on the CPU).
#pragma once
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include "fft16.cuh"

namespace ssb {

namespace cg = cooperative_groups;

constexpr int C64_LOG2M = 16;
constexpr int C64_M = 1 << C64_LOG2M;
constexpr int C64_NS = 4096;                       // sub-transform size
constexpr int C64_TPB = 1024;                      // 4 groups x 256 threads
constexpr int C64_CL = 4;                          // CTAs per cluster
constexpr int C64_BUF = FftPlan<12>::SMEM_ELEMS;   // float2 per group buffer (4096 + padding)
constexpr int C64_SMEM_BYTES = 4 * C64_BUF * (int)sizeof(float2);
constexpr int C64_TWM_ELEMS = 16 * 1024;           // TWM[r][tau] = w_M^(tau r)

__constant__ float2 kW64[64];                      // w_64^k = exp(-2 pi i k / 64), correctly rounded

struct GroupBar {                                  // named barrier of one 256-thread group (ids 1..4; 0 = __syncthreads)
    int id;
    __device__ __forceinline__ void operator()() const { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }
};

// multiply by (-i)^k (forward w4^k), k in 0..3, k uniform
__device__ __forceinline__ float2 rot_fwd(float2 a, int k) {
    switch (k & 3) {
        case 1: return make_float2(a.y, -a.x);
        case 2: return make_float2(-a.x, -a.y);
        case 3: return make_float2(-a.y, a.x);
        default: return a;
    }
}

// xs[j] = x_ext[m0 - D + j]: zeros before the clip, one wrap past its end when `wrap` (continuous_simulator.py:440-445)
__device__ __forceinline__ float src_sample(const float* __restrict__ src, int S, long long n, int wrap) {
    if (n < 0) return 0.f;
    if (n < S) return __ldg(src + n);
    if (wrap && n - S < S) return __ldg(src + (n - S));
    return 0.f;
}

// Source spectrum SX[r][slot]: grid (16), block 256, dynamic smem C64_BUF float2.
__global__ void __launch_bounds__(256)
src64k_kernel(const float* __restrict__ src, int S, long long m0, int wrap, int D, float2* __restrict__ SX,
              const float2* __restrict__ tw12, const float2* __restrict__ twm) {
    using P = FftPlan<12>;
    extern __shared__ float2 smem[];
    const int r = blockIdx.x, t = threadIdx.x;
    const Tw6 w0 = load_tw6<true>(tw12, P::T, t);
    float2 v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int n1 = t + 256 * j;
        float2 acc = make_float2(0.f, 0.f);
#pragma unroll 4
        for (int q = 0; q < 16; ++q) {
            const float x = src_sample(src, S, m0 - D + n1 + C64_NS * q, wrap);
            const float2 w = kW64[(4 * q * r) & 63];                       // w16^(q r)
            acc = fma2(bcast(x), w, acc);
        }
        const float2 tw = cmul(__ldg(twm + r * 1024 + (n1 & 1023)), kW64[((n1 >> 10) * r) & 63]);   // w_M^(n1 r)
        v[j] = cmul(acc, tw);
    }
    fft_forward<12>(v, t, smem, w0, tw12 + P::TW_SMALL_OFFSET);
#pragma unroll
    for (int i = 0; i < 16; ++i) SX[(long long)r * C64_NS + i * P::T + t] = v[i];
}

// grid (4 * B), cluster (4,1,1), block C64_TPB, dynamic smem C64_SMEM_BYTES.
// The CTA's four sub-problems are transformed side by side, one per 256-thread group (1024 threads, the whole register
// file of the SM).  In the staging phases (A, E, F) thread tau = threadIdx.x handles n1 = tau + 1024 i, i = 0..3.
__global__ void __cluster_dims__(C64_CL, 1, 1) __launch_bounds__(C64_TPB, 1)
conv64k_kernel(const ssb_req* __restrict__ reqs, const float2* __restrict__ rir_bank, const float2* __restrict__ xpool,
               float* __restrict__ wave, long long wave_stride, int sr, const float2* __restrict__ tw12,
               const float2* __restrict__ twm) {
    using P = FftPlan<12>;
    extern __shared__ float2 smem[];
    cg::cluster_group cluster = cg::this_cluster();
    const int c = (int)cluster.block_rank();            // residue class of the spectrum bins this CTA owns
    const int env = blockIdx.x / C64_CL;
    const int tau = threadIdx.x;                        // 0..1023
    const int t = threadIdx.x & 255;                    // thread within its group
    const int grp = threadIdx.x >> 8;
    const ssb_req& rq = reqs[env];
    const int taps = (rq.flags & SSB_FLAG_SILENT) ? 0 : rq.term[0].rir_taps;
    const int nvalid = taps > 0 ? min(rq.out_samples, sr) : 0;
    const int D = C64_M - sr;
    float* __restrict__ wl = wave + (long long)env * 2 * wave_stride;
    float* __restrict__ wr = wl + wave_stride;
    if (nvalid == 0) {                                  // silent / zero RIR: exact zeros (cluster-uniform exit)
        for (int n = c * C64_TPB + tau; n < sr; n += C64_CL * C64_TPB) { wl[n] = 0.f; wr[n] = 0.f; }
        return;
    }
    // ---- phase A: modulate by the residue class, radix-4 over q1 (and q2 for taps > 16384), twiddle -> a_r[n1]
    {
        float2 twr[4];                                  // w_M^(tau r), r = c + 4 m' (re-read in phase E: 8 registers less across the transforms)
#pragma unroll
        for (int mm = 0; mm < 4; ++mm) twr[mm] = __ldg(twm + (c + 4 * mm) * 1024 + tau);
        const float2* __restrict__ h = rir_bank + rq.term[0].rir_offset;
        const int nq2 = (taps + 16383) >> 14;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int n1 = tau + 1024 * i;
            float2 u[4];
#pragma unroll
            for (int q1 = 0; q1 < 4; ++q1) {
                const int n = n1 + C64_NS * q1;
                u[q1] = n < taps ? __ldg(h + n) : make_float2(0.f, 0.f);
            }
            for (int q2 = 1; q2 < nq2; ++q2) {                              // rare: RIR longer than 16384 taps
#pragma unroll
                for (int q1 = 0; q1 < 4; ++q1) {
                    const int n = n1 + C64_NS * (q1 + 4 * q2);
                    const float2 x = n < taps ? __ldg(h + n) : make_float2(0.f, 0.f);
                    u[q1] = add2(u[q1], rot_fwd(x, q2 * c));
                }
            }
            if (c != 0) {
#pragma unroll
                for (int q1 = 0; q1 < 4; ++q1) u[q1] = cmul(u[q1], kW64[((4 * q1 + i) * c) & 63]);   // w16^(q1 c) w64^(i c)
            }
            bfly4<false>(u[0], u[1], u[2], u[3]);                           // u[m'] = sum_q1 w4^(q1 m') u[q1]
            // x w_M^(tau r) w16^(i m')
            smem[0 * C64_BUF + n1] = cmul(u[0], twr[0]);
            if (i == 0) {
                smem[1 * C64_BUF + n1] = cmul(u[1], twr[1]);
                smem[2 * C64_BUF + n1] = cmul(u[2], twr[2]);
                smem[3 * C64_BUF + n1] = cmul(u[3], twr[3]);
            } else if (i == 1) {
                smem[1 * C64_BUF + n1] = cmul(mul_w16<false, 1>(u[1]), twr[1]);
                smem[2 * C64_BUF + n1] = cmul(mul_w16<false, 2>(u[2]), twr[2]);
                smem[3 * C64_BUF + n1] = cmul(mul_w16<false, 3>(u[3]), twr[3]);
            } else if (i == 2) {
                smem[1 * C64_BUF + n1] = cmul(mul_w16<false, 2>(u[1]), twr[1]);
                smem[2 * C64_BUF + n1] = cmul(mul_w16<false, 4>(u[2]), twr[2]);
                smem[3 * C64_BUF + n1] = cmul(mul_w16<false, 6>(u[3]), twr[3]);
            } else {
                smem[1 * C64_BUF + n1] = cmul(mul_w16<false, 3>(u[1]), twr[1]);
                smem[2 * C64_BUF + n1] = cmul(mul_w16<false, 6>(u[2]), twr[2]);
                smem[3 * C64_BUF + n1] = cmul(mul_w16<false, 9>(u[3]), twr[3]);
            }
        }
    }
    __syncthreads();

    // ---- phases B-D: group grp transforms sub-problem r = c + 4 grp, multiplies by the source spectrum, transforms back
    {
        float2* __restrict__ buf = smem + grp * C64_BUF;
        const GroupBar bar{1 + grp};
        const int r = c + 4 * grp;
        float2 v[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = buf[t + 256 * j];
        const Tw6 w0 = load_tw6<true>(tw12, P::T, t);
        bar();                                                              // inputs read before the exchange overwrites them
        fft_forward<12>(v, t, buf, w0, tw12 + P::TW_SMALL_OFFSET, bar);
        const float2* __restrict__ sx = xpool + rq.term[0].x_offset + (long long)r * C64_NS + t;
#pragma unroll
        for (int i0 = 0; i0 < 16; i0 += 4) {                                // 4 at a time: 64 registers per thread in all
            float2 s[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) s[i] = __ldg(sx + (i0 + i) * P::T);
#pragma unroll
            for (int i = 0; i < 4; ++i) v[i0 + i] = cmul(v[i0 + i], s[i]);
        }
        bar();                                                              // the forward's last exchange reads are done
        fft_inverse<12, true>(v, t, buf, tw12, tw12 + P::TW_SMALL_OFFSET, bar);
        bar();                                                              // the inverse's last exchange reads are done
#pragma unroll
        for (int j = 0; j < 16; ++j) buf[t + 256 * j] = v[j];               // e_r[n1], n1 = t + 256 j (unscaled)
    }
    __syncthreads();

    // ---- phase E: conj twiddle, inverse radix-4 over m', demodulate; in place: buffer q1 <- v_c[q1][n1]
    {
        float2 twr[4];
#pragma unroll
        for (int mm = 0; mm < 4; ++mm) twr[mm] = __ldg(twm + (c + 4 * mm) * 1024 + tau);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int n1 = tau + 1024 * i;
            float2 b[4];
            b[0] = cmulc(smem[0 * C64_BUF + n1], twr[0]);
            if (i == 0) {
                b[1] = cmulc(smem[1 * C64_BUF + n1], twr[1]);
                b[2] = cmulc(smem[2 * C64_BUF + n1], twr[2]);
                b[3] = cmulc(smem[3 * C64_BUF + n1], twr[3]);
            } else if (i == 1) {
                b[1] = mul_w16<true, 1>(cmulc(smem[1 * C64_BUF + n1], twr[1]));
                b[2] = mul_w16<true, 2>(cmulc(smem[2 * C64_BUF + n1], twr[2]));
                b[3] = mul_w16<true, 3>(cmulc(smem[3 * C64_BUF + n1], twr[3]));
            } else if (i == 2) {
                b[1] = mul_w16<true, 2>(cmulc(smem[1 * C64_BUF + n1], twr[1]));
                b[2] = mul_w16<true, 4>(cmulc(smem[2 * C64_BUF + n1], twr[2]));
                b[3] = mul_w16<true, 6>(cmulc(smem[3 * C64_BUF + n1], twr[3]));
            } else {
                b[1] = mul_w16<true, 3>(cmulc(smem[1 * C64_BUF + n1], twr[1]));
                b[2] = mul_w16<true, 6>(cmulc(smem[2 * C64_BUF + n1], twr[2]));
                b[3] = mul_w16<true, 9>(cmulc(smem[3 * C64_BUF + n1], twr[3]));
            }
            bfly4<true>(b[0], b[1], b[2], b[3]);                            // b[q1] = sum_m' conj(w4)^(q1 m') b[m']
            if (c != 0) {
#pragma unroll
                for (int q1 = 0; q1 < 4; ++q1) b[q1] = cmulc(b[q1], kW64[((4 * q1 + i) * c) & 63]);
            }
#pragma unroll
            for (int q1 = 0; q1 < 4; ++q1) smem[q1 * C64_BUF + n1] = b[q1];
        }
    }
    cluster.sync();

    // ---- phase F: CTA k combines n1 in [1024 k, 1024 k + 1024): radix-4 over the CTAs through distributed shared memory
    {
        const float2* __restrict__ peer[C64_CL];
#pragma unroll
        for (int cc = 0; cc < C64_CL; ++cc) peer[cc] = cluster.map_shared_rank(smem, cc);
        constexpr float scale = 1.0f / (float)C64_M;
        const int n1 = C64_TPB * c + tau;
        float2 val[4][4];
#pragma unroll
        for (int q1 = 0; q1 < 4; ++q1)
#pragma unroll
            for (int cc = 0; cc < C64_CL; ++cc) val[q1][cc] = peer[cc][q1 * C64_BUF + n1];
#pragma unroll
        for (int q1 = 0; q1 < 4; ++q1) {
            bfly4<true>(val[q1][0], val[q1][1], val[q1][2], val[q1][3]);        // val[q1][q2] = sum_c conj(w4)^(q2 c) v_c
#pragma unroll
            for (int q2 = 0; q2 < 4; ++q2) {
                const int mo = n1 + C64_NS * (q1 + 4 * q2) - D;                 // output sample index
                if (mo >= 0 && mo < sr) {
                    const bool ok = mo < nvalid;
                    wl[mo] = ok ? val[q1][q2].x * scale : 0.f;
                    wr[mo] = ok ? val[q1][q2].y * scale : 0.f;
                }
            }
        }
    }
    cluster.sync();                                                         // peers may still be reading this CTA's buffers
}

}  // namespace ssb
