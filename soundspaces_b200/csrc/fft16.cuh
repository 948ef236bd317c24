// Register-resident radix-16 FFT for sm_90a.
//
// One "group" of T = N/16 threads transforms N = 2^LOG2N complex points; every
// thread keeps 16 points in registers for the whole transform.  A transform is
//   NPASS = LOG2N/4 radix-16 passes (4x4 butterflies in registers), with one
//   shared-memory exchange between consecutive passes, followed by
//   a radix-M stage (M = N / 16^NPASS in {1,2,4}) done with warp shuffles
//   between M adjacent lanes.
// The forward transform is decimation-in-frequency and leaves the spectrum in
// a fixed digit-permuted order ("slot order": slot = i*T + t for register i of
// thread t); the inverse transform is the exact mirror image (decimation in
// time) and consumes slot order, so the pointwise spectrum product of the
// overlap-save convolution never needs a reordering pass.  freq_of_slot()
// gives the permutation for callers that need natural order (the STFT).
//
// Twiddles: the 15 inter-pass twiddles w^(j s), s = r + 4m, are applied in two
// factors inside the 4x4 butterfly -- w^(j r) between the two radix-4 stages and
// w^(4 j m) after the second -- so a thread needs only SIX correctly rounded table
// entries per pass (w^j, w^2j, w^3j, w^4j, w^8j, w^12j) instead of fifteen.  Pass 0
// (stride T: one distinct set per thread) is read from global memory early by the
// caller; the later passes (stride <= 64) come from a small table staged in shared
// memory.  (A product tree from w^1 alone is cheaper still but its 3-4 ulp error
// leaks the loudest bin into quiet ones: 8x the error on music, DESIGN.md "Numerics".)
//
// Exchanges: one padding rule per transform size keeps every access pattern
// bank-conflict free and makes the region a group of stride(p-1) threads touches in
// the exchange before pass p private to that group, so exchanges whose group is one
// warp only need __syncwarp().
//
// No cuFFT, no library code: this is the hot loop of the SoundSpaces audio
// path (scipy.signal.fftconvolve at soundspaces/simulator.py:630-647 and
// librosa.stft at soundspaces/tasks/nav.py:92 in the reference).
#pragma once
#include <cuda_runtime.h>

namespace ssb {

// ---------------------------------------------------------------------------------------------
// Complex arithmetic on FP32 pairs, one scalar FADD / FMUL / FFMA per half (sm_90a has no two-wide
// FP32 instructions).  The _rn intrinsics pin each half to one correctly rounded operation, so ptxas
// never contracts a product and a sum into an FMA of its own choosing: every result is the same
// bit pattern whichever way the pair is scheduled.  Multiplying by +-i is a pure operand swizzle.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 sub2(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 bcast(float x) { return make_float2(x, x); }

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return add2(a, b); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return sub2(a, b); }
// a * b = a.x * (b.x, b.y) + a.y * (-b.y, b.x)          (2 FMUL + 2 FFMA)
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
    const float2 t = mul2(bcast(a.y), make_float2(b.y, b.x));
    return fma2(bcast(a.x), b, make_float2(-t.x, t.y));
}
// a * conj(b) = a.x * (b.x, -b.y) + a.y * (b.y, b.x)
__device__ __forceinline__ float2 cmulc(float2 a, float2 b) {
    const float2 t = mul2(bcast(a.y), make_float2(b.y, b.x));
    return fma2(bcast(a.x), make_float2(b.x, -b.y), t);
}
// acc + a * b   (2 FFMA + 2 FMUL + 2 FADD: the half-negation folds into the add's operand modifier)
__device__ __forceinline__ float2 cfma(float2 a, float2 b, float2 acc) {
    const float2 t = mul2(bcast(a.y), make_float2(b.y, b.x));
    return add2(fma2(bcast(a.x), b, acc), make_float2(-t.x, t.y));
}
// a * (-i) and a * (+i): pure operand swizzles
__device__ __forceinline__ float2 mul_mi(float2 a) { return make_float2(a.y, -a.x); }
__device__ __forceinline__ float2 mul_pi(float2 a) { return make_float2(-a.y, a.x); }

// 4-point DFT, in place.  Forward: w4 = -i.  Inverse: w4 = +i.   (16 FADD)
template <bool INV>
__device__ __forceinline__ void bfly4(float2& a0, float2& a1, float2& a2, float2& a3) {
    float2 t0 = cadd(a0, a2), t1 = csub(a0, a2), t2 = cadd(a1, a3), t3 = csub(a1, a3);
    float2 r = INV ? mul_pi(t3) : mul_mi(t3);
    a0 = cadd(t0, t2);
    a2 = csub(t0, t2);
    a1 = cadd(t1, r);
    a3 = csub(t1, r);
}

// multiply by w16^k (forward) or conj(w16^k) (inverse), k a compile-time constant
template <bool INV, int K>
__device__ __forceinline__ float2 mul_w16(float2 a) {
    constexpr float C1 = 0.92387953251128674f;   // cos(pi/8)
    constexpr float S1 = 0.38268343236508977f;   // sin(pi/8)
    constexpr float R2 = 0.70710678118654752f;
    static_assert(K == 0 || K == 1 || K == 2 || K == 3 || K == 4 || K == 6 || K == 9, "unsupported w16 power");
    // forward twiddle w16^k = cos(k pi/8) - i sin(k pi/8); the inverse uses the conjugate
    if constexpr (K == 0) return a;
    else if constexpr (K == 1) return cmul(a, make_float2(C1, INV ? S1 : -S1));
    else if constexpr (K == 2)                   // R2 (1 -+ i) a = R2 (a + (-+i) a)
        return mul2(cadd(a, INV ? mul_pi(a) : mul_mi(a)), bcast(R2));
    else if constexpr (K == 3) return cmul(a, make_float2(S1, INV ? C1 : -C1));
    else if constexpr (K == 4) return INV ? mul_pi(a) : mul_mi(a);
    else if constexpr (K == 6)                   // R2 (-1 -+ i) a = R2 ((-+i) a - a)
        return mul2(csub(INV ? mul_pi(a) : mul_mi(a), a), bcast(R2));
    else return cmul(a, make_float2(-C1, INV ? -S1 : S1));   // K == 9
}

// the six inter-pass twiddles of one thread for one pass: r[k-1] = w^(j k), m[k-1] = w^(4 j k), k = 1..3
struct Tw6 {
    float2 r[3];
    float2 m[3];
};

// table rows [6][st]: w^j, w^2j, w^3j, w^4j, w^8j, w^12j with w = exp(-2 pi i / (16 st)); tab points at column 0
template <bool GLOBAL>
__device__ __forceinline__ Tw6 load_tw6(const float2* __restrict__ tab, int st, int j) {
    Tw6 w;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        w.r[k] = GLOBAL ? __ldg(tab + k * st + j) : tab[k * st + j];
        w.m[k] = GLOBAL ? __ldg(tab + (3 + k) * st + j) : tab[(3 + k) * st + j];
    }
    return w;
}

// 16-point DFT in registers with the inter-pass twiddles folded in.
//   forward (DIF):  v[s] <- w^(j s) * sum_q v[q] w16^(q s)
//   inverse (DIT):  v[q] <- sum_s conj(w^(j s)) v[s] conj(w16)^(q s)
// TW = false skips the inter-pass twiddles (stride-1 pass: j == 0 for every thread).
template <bool INV, bool TW>
__device__ __forceinline__ void fft16(float2 (&v)[16], const Tw6& w) {
    if constexpr (INV && TW) {
        // input s = r + 4m sits in v[s]; undo w^(4 j m)
#pragma unroll
        for (int m = 1; m < 4; ++m)
#pragma unroll
            for (int r = 0; r < 4; ++r) v[r + 4 * m] = cmulc(v[r + 4 * m], w.m[m - 1]);
    }
    // stage 1: 4-point DFTs over q = c + 4d (d = 0..3); result a[c][r] left in v[c + 4r]
#pragma unroll
    for (int c = 0; c < 4; ++c) bfly4<INV>(v[c], v[c + 4], v[c + 8], v[c + 12]);
    // twiddles w16^(c r)
    v[5] = mul_w16<INV, 1>(v[5]);
    v[9] = mul_w16<INV, 2>(v[9]);
    v[13] = mul_w16<INV, 3>(v[13]);
    v[6] = mul_w16<INV, 2>(v[6]);
    v[10] = mul_w16<INV, 4>(v[10]);
    v[14] = mul_w16<INV, 6>(v[14]);
    v[7] = mul_w16<INV, 3>(v[7]);
    v[11] = mul_w16<INV, 6>(v[11]);
    v[15] = mul_w16<INV, 9>(v[15]);
    if constexpr (TW) {
        if constexpr (!INV) {
            // forward: a[c][r] (in v[c + 4r]) *= w^(j r)
#pragma unroll
            for (int r = 1; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) v[c + 4 * r] = cmul(v[c + 4 * r], w.r[r - 1]);
        } else {
            // inverse: element (c' = the forward's r, r') in v[c' + 4r'] *= conj(w^(j c'))
#pragma unroll
            for (int c = 1; c < 4; ++c)
#pragma unroll
                for (int r = 0; r < 4; ++r) v[c + 4 * r] = cmulc(v[c + 4 * r], w.r[c - 1]);
        }
    }
    // stage 2: 4-point DFTs over c for each r; output s = r + 4m is left in v[4r + m]
#pragma unroll
    for (int r = 0; r < 4; ++r) bfly4<INV>(v[4 * r], v[4 * r + 1], v[4 * r + 2], v[4 * r + 3]);
    if constexpr (TW && !INV) {
        // forward: X[r + 4m] (in v[4r + m]) *= w^(4 j m)
#pragma unroll
        for (int m = 1; m < 4; ++m)
#pragma unroll
            for (int r = 0; r < 4; ++r) v[4 * r + m] = cmul(v[4 * r + m], w.m[m - 1]);
    }
    // un-transpose: out[s] = v[4*(s%4) + s/4]
    float2 u[16];
#pragma unroll
    for (int s = 0; s < 16; ++s) u[s] = v[4 * (s & 3) + (s >> 2)];
#pragma unroll
    for (int s = 0; s < 16; ++s) v[s] = u[s];
}

template <int LOG2N>
struct FftPlan {
    static constexpr int N = 1 << LOG2N;
    static constexpr int T = N / 16;                       // threads per transform
    static constexpr int NPASS = LOG2N / 4;                // radix-16 passes
    static constexpr int M = N >> (4 * NPASS);             // leftover radix (lanes)
    static_assert(M == 1 || M == 2 || M == 4, "supported sizes: 2^{8,9,10,12,13,14}");
    static_assert(T >= 32 || T == 16, "group must be whole warps");
    __host__ __device__ static constexpr int stride(int p) { return N >> (4 * (p + 1)); }
    // exchange-buffer padding: PADST float2 after every 16*PADST elements, PADST = stride of the
    // last pass (none needed when that is >= 16)
    static constexpr int PADST = stride(NPASS - 1) >= 16 ? 0 : stride(NPASS - 1);
    // shared memory (float2 elements) for the exchange buffer, with padding
    static constexpr int SMEM_ELEMS = N + N / 16;
    // twiddle table: pass p occupies 6 * stride(p) float2 at tw_offset(p), rows
    // exp(-2 pi i * j * e / (16 * stride(p))) for e in {1, 2, 3, 4, 8, 12}, j < stride(p)
    __host__ __device__ static constexpr int tw_offset(int p) {
        int o = 0;
        for (int q = 0; q < p; ++q) o += 6 * stride(q);
        return o;
    }
    static constexpr int TW_ELEMS = tw_offset(NPASS);
    // passes >= 1 ("small" table, staged in shared memory by the kernels)
    static constexpr int TW_SMALL_OFFSET = tw_offset(1);
    static constexpr int TW_SMALL_ELEMS = TW_ELEMS - TW_SMALL_OFFSET;
};

// logical element index held by thread t, register i during pass with stride st
__device__ __forceinline__ int pass_pos(int t, int i, int st) {
    return (t / st) * (16 * st) + (t % st) + i * st;
}
template <int PADST>
__device__ __forceinline__ int pad_idx(int l) {
    if constexpr (PADST == 0) return l;
    else return l + PADST * (l / (16 * PADST));
}
// pad_idx(pass_pos(t, i, st)) is affine in i: base + i * stride with a compile-time stride, so the 16
// exchange accesses of a pass use one computed address plus immediates.  (For st >= 16*PADST the i*st term
// is a whole number of padding periods; the last pass has st == PADST and its 16 elements share one period.)
template <int PADST>
__device__ __forceinline__ int pass_base(int t, int st) { return pad_idx<PADST>(pass_pos(t, 0, st)); }
template <int PADST>
__host__ __device__ constexpr int pass_stride(int st) {
    return (PADST > 0 && st >= 16 * PADST) ? st + st / 16 : st;
}

// barrier among the G consecutive threads that share an exchange region
template <int G>
__device__ __forceinline__ void group_barrier() {
    if constexpr (G <= 32) __syncwarp();
    else __syncthreads();                                  // G > 32 only occurs with group == CTA (or 2 warps of it)
}

// barrier among the threads of one transform when they span more than a warp: the whole CTA by default; kernels
// that run several transforms side by side in one CTA pass a named barrier of their group (conv64k.cuh)
struct CtaBar {
    __device__ __forceinline__ void operator()() const { __syncthreads(); }
};

// Forward transform.  In: v[q] = x[t + q*T].  Out: v[i] = spectrum slot (t, i).
// w0: pass-0 twiddles of this thread (load_tw6 at column t of the pass-0 table), loaded by the
//     caller so the loads can be issued early.
// stw: table of passes >= 1 (pass p at FftPlan::tw_offset(p) - TW_SMALL_OFFSET), normally in shared memory.
// buf: >= SMEM_ELEMS float2, private to the group; the caller orders other uses of buf.
// LANE_STAGE = false leaves out the final radix-M stage across lanes: the caller folds it into its own
// reads (the STFT kernel does, for M = 2: lane 2a then holds P_a[i], lane 2a+1 holds Q_a[i], and
// X[a + 16 i] = P + Q, X[a + 16 i + N/2] = P - Q).
// twp(p, st) returns this thread's twiddles of pass p >= 1 (stride st > 1).
template <int LOG2N, bool LANE_STAGE, class Bar, class TwP>
__device__ __forceinline__ void fft_forward_impl(float2 (&v)[16], int t, float2* __restrict__ buf, const Tw6& w0,
                                                 const TwP& twp, const Bar bar) {
    using P = FftPlan<LOG2N>;
    fft16<false, true>(v, w0);
#pragma unroll
    for (int p = 1; p < P::NPASS; ++p) {
        const int st = P::stride(p), stp = P::stride(p - 1);
        // exchange: written with pass p-1 layout, read with pass p layout; shared by stp threads
        if (p > 1) { if (stp <= 32) __syncwarp(); else bar(); }      // previous readers of this region
        {
            float2* __restrict__ wp = buf + pass_base<P::PADST>(t, stp);
#pragma unroll
            for (int i = 0; i < 16; ++i) wp[i * pass_stride<P::PADST>(P::stride(p - 1))] = v[i];
        }
        if (stp <= 32) __syncwarp(); else bar();
        {
            const float2* __restrict__ rp = buf + pass_base<P::PADST>(t, st);
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] = rp[i * pass_stride<P::PADST>(P::stride(p))];
        }
        if (st > 1) {
            fft16<false, true>(v, twp(p, st));
        } else {
            fft16<false, false>(v, w0);
        }
    }
    // leftover radix-M across M adjacent lanes (DIF)
    if constexpr (!LANE_STAGE) {
        return;
    } else if constexpr (P::M == 2) {
        const float sgn = (t & 1) ? -1.f : 1.f;                // lower lane: v + o, upper lane: o - v  (one FFMA each)
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            float2 o = make_float2(__shfl_xor_sync(0xffffffffu, v[i].x, 1), __shfl_xor_sync(0xffffffffu, v[i].y, 1));
            v[i] = fma2(bcast(sgn), v[i], o);
        }
    } else if constexpr (P::M == 4) {
        const int j = t & 3;
        const bool up2 = j & 2, up1 = j & 1;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            float2 o = make_float2(__shfl_xor_sync(0xffffffffu, v[i].x, 2), __shfl_xor_sync(0xffffffffu, v[i].y, 2));
            float2 r = up2 ? csub(o, v[i]) : cadd(v[i], o);
            if (j == 3) r = mul_mi(r);                     // (a0 - a1) * w4^1
            o = make_float2(__shfl_xor_sync(0xffffffffu, r.x, 1), __shfl_xor_sync(0xffffffffu, r.y, 1));
            v[i] = up1 ? csub(o, r) : cadd(r, o);
        }
    }
}

template <int LOG2N, bool LANE_STAGE = true, class Bar = CtaBar>
__device__ __forceinline__ void fft_forward(float2 (&v)[16], int t, float2* __restrict__ buf, const Tw6& w0,
                                            const float2* __restrict__ stw, const Bar bar = Bar()) {
    using P = FftPlan<LOG2N>;
    fft_forward_impl<LOG2N, LANE_STAGE>(v, t, buf, w0, [&](int p, int st) {
        return load_tw6<false>(stw + (P::tw_offset(p) - P::TW_SMALL_OFFSET), st, t % st);
    }, bar);
}

// Two-pass sizes (N = 512, 1024): w1 holds this thread's pass-1 twiddles (load_tw6 at column t % stride(1) of the
// pass-1 table), loaded by the caller -- once for a whole loop of transforms, like w0.
template <int LOG2N, bool LANE_STAGE = true, class Bar = CtaBar>
__device__ __forceinline__ void fft_forward(float2 (&v)[16], int t, float2* __restrict__ buf, const Tw6& w0,
                                            const Tw6& w1, const Bar bar = Bar()) {
    static_assert(FftPlan<LOG2N>::NPASS == 2, "w1 is the twiddle set of the only later pass");
    fft_forward_impl<LOG2N, LANE_STAGE>(v, t, buf, w0, [&](int, int) -> const Tw6& { return w1; }, bar);
}

// Inverse transform (unscaled).  In: v[i] = spectrum slot (t, i).  Out: v[q] = N * x[t + q*T].
// gtw0: pass-0 table (column 0; global memory when TW0_GLOBAL); its six entries are fetched before
// the last exchange so the latency overlaps it.  stw: as for fft_forward.
template <int LOG2N, bool TW0_GLOBAL = true, class Bar = CtaBar>
__device__ __forceinline__ void fft_inverse(float2 (&v)[16], int t, float2* __restrict__ buf,
                                            const float2* __restrict__ gtw0, const float2* __restrict__ stw,
                                            const Bar bar = Bar()) {
    using P = FftPlan<LOG2N>;
    if constexpr (P::M == 2) {
        const float sgn = (t & 1) ? -1.f : 1.f;                // lower lane: v + o, upper lane: o - v  (one FFMA each)
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            float2 o = make_float2(__shfl_xor_sync(0xffffffffu, v[i].x, 1), __shfl_xor_sync(0xffffffffu, v[i].y, 1));
            v[i] = fma2(bcast(sgn), v[i], o);
        }
    } else if constexpr (P::M == 4) {
        const int j = t & 3;
        const bool up2 = j & 2, up1 = j & 1;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            float2 o = make_float2(__shfl_xor_sync(0xffffffffu, v[i].x, 1), __shfl_xor_sync(0xffffffffu, v[i].y, 1));
            float2 r = up1 ? csub(o, v[i]) : cadd(v[i], o);
            if (j == 3) r = mul_pi(r);                     // * conj(w4^1)
            o = make_float2(__shfl_xor_sync(0xffffffffu, r.x, 2), __shfl_xor_sync(0xffffffffu, r.y, 2));
            v[i] = up2 ? csub(o, r) : cadd(r, o);
        }
    }
    Tw6 w0;
    if constexpr (P::NPASS == 1) w0 = load_tw6<TW0_GLOBAL>(gtw0, P::stride(0), t);
#pragma unroll
    for (int p = P::NPASS - 1; p >= 1; --p) {
        const int st = P::stride(p), stn = P::stride(p - 1);
        if (st > 1) {
            const Tw6 w = load_tw6<false>(stw + (P::tw_offset(p) - P::TW_SMALL_OFFSET), st, t % st);
            fft16<true, true>(v, w);
        } else {
            fft16<true, false>(v, w0);
        }
        if (p == 1) w0 = load_tw6<TW0_GLOBAL>(gtw0, P::stride(0), t);      // in flight during the exchange
        // exchange: written with pass p layout, read with pass p-1 layout; shared by stn threads.
        // The region was last read (previous exchange) by this thread's st-group only.
        if (p < P::NPASS - 1) { if (st <= 32) __syncwarp(); else bar(); }
        {
            float2* __restrict__ wp = buf + pass_base<P::PADST>(t, st);
#pragma unroll
            for (int i = 0; i < 16; ++i) wp[i * pass_stride<P::PADST>(P::stride(p))] = v[i];
        }
        if (stn <= 32) __syncwarp(); else bar();
        {
            const float2* __restrict__ rp = buf + pass_base<P::PADST>(t, stn);
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] = rp[i * pass_stride<P::PADST>(P::stride(p - 1))];
        }
    }
    fft16<true, true>(v, w0);
}

// frequency index of spectrum slot (thread t, register i)
template <int LOG2N>
__host__ __device__ inline int freq_of_slot(int t, int i) {
    using P = FftPlan<LOG2N>;
    // position after the last radix-16 pass
    int pos = (t / P::stride(P::NPASS - 1)) * (16 * P::stride(P::NPASS - 1)) + (t % P::stride(P::NPASS - 1)) +
              i * P::stride(P::NPASS - 1);
    int k = 0, mult = 1, rem = pos;
    for (int p = 0; p < P::NPASS; ++p) {
        int st = P::stride(p);
        k += (rem / st) * mult;
        rem %= st;
        mult *= 16;
    }
    if (P::M == 2) k += rem * mult;
    if (P::M == 4) k += (((rem & 1) << 1) | (rem >> 1)) * mult;
    return k;
}

}  // namespace ssb
