// kernels_simt.cuh -- CUDA-core kernels of the RNN-T loss hot path (sm_90a).
//
//   lse_gather_kernel   log-softmax denominators + (blank, label) log-prob gather, one pass
//                       (replaces reduce_max + reduce_exp + logp(): gpu_rnnt.h:73-80,
//                        reduce.h:45-104, gpu_rnnt_kernel.h:5-9)
//   alpha_beta_kernel   forward/backward lattice recurrences as anti-diagonal wavefronts over a
//                       DIAGONAL-MAJOR cache of the two log-probs per cell
//                       (replaces gpu_rnnt_kernel.h:11-47, 79-113; arithmetic of cpu_rnnt.h:175-253)
//   rnnt_grad_kernel    gradient w.r.t. logits (gpu_rnnt_kernel.h:143-179), padded cells zeroed
//                       in the same pass (replaces the cudaMemsetAsync of gpu_rnnt.h:109)
//   alpha_beta_windowed_kernel   the same wavefronts under the alignment-restricted loss's per-column frame windows
//                       (struct Windows); lse_gather, rnnt_grad and row_scale take the windows too
//   row_scale_kernel    per-row scales of the tensor-core backward GEMMs + the patch of the two special columns
//   zgen/sgemm/...      fp32 building blocks of the exact (RNNTB200_FP32_EXACT) joint path, and colsum (also dense1's db1)
// lse_gather and rnnt_grad also take fp16 / bf16 logits (and write gradients of that type) over fp32 arithmetic; their
// scalar and 16-byte (_vec) kernels share row_cell (and store_lse_logprobs); arc_terms serves rnnt_grad[_vec] and row_scale.
//
// Data layout ("skewed" planes): a per-utterance plane stores cell (t,u) at row n=t+u, column u:
//     sk(b,t,u) = b*SK + (t+u)*maxU + u,   SK = (maxT+maxU-1)*maxU
// so that step n of a wavefront touches ONE contiguous row (coalesced), which the reference's
// (t*maxU+u) planes cannot offer (stride maxU-1 between neighbouring threads).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

namespace rb {

template <typename T> __device__ __forceinline__ T neg_inf();
template <> __device__ __forceinline__ float neg_inf<float>() { return -CUDART_INF_F; }
template <> __device__ __forceinline__ double neg_inf<double>() { return -CUDART_INF; }

__device__ __forceinline__ float  xexp(float x)    { return expf(x); }
__device__ __forceinline__ double xexp(double x)   { return exp(x); }
__device__ __forceinline__ float  xlog(float x)    { return logf(x); }
__device__ __forceinline__ double xlog(double x)   { return log(x); }
__device__ __forceinline__ float  xlog1p(float x)  { return log1pf(x); }
__device__ __forceinline__ double xlog1p(double x) { return log1p(x); }

// rnnt_helper::log_sum_exp -- rnnt_helper.h:16-24 (including the -inf short circuits)
template <typename T>
__device__ __forceinline__ T log_sum_exp(T a, T b) {
    if (a == neg_inf<T>()) return b;
    if (b == neg_inf<T>()) return a;
    return a > b ? xlog1p(xexp(b - a)) + a : xlog1p(xexp(a - b)) + b;
}

// Wavefront variant for float: the recurrence is a chain of T+U-1 DEPENDENT log-sum-exps, so its latency (not its
// throughput) sets the kernel time.  max + log2(1 + 2^(-|a-b|*log2 e)) * ln 2 on the MUFU ex2/lg2 units is ~3x
// shorter than log1pf(expf(.)) and agrees with it to a few ulp (|error| < 3e-7 per step, far inside rtol 1e-4).
__device__ __forceinline__ float log_sum_exp_fast(float a, float b) {
    // branch-free (the chain's latency is what counts): with one argument -inf the exponential is 0 and the result the other
    // argument, bit for bit (lg2(1) = 0); with both -inf the difference is forced to 0 and the result is -inf + ln 2 = -inf
    const float mx = fmaxf(a, b), mn = fminf(a, b);
    const float d = (mx == -CUDART_INF_F) ? 0.f : mn - mx;
    float e, l;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(d * 1.4426950408889634f));
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(1.f + e));
    return fmaf(l, 0.6931471805599453f, mx);
}
__device__ __forceinline__ float  wave_lse(float a, float b)  { return log_sum_exp_fast(a, b); }
__device__ __forceinline__ double wave_lse(double a, double b) { return log_sum_exp<double>(a, b); }

// Element types of the loss op's logits and gradients (X) next to its workspace type (T = float or double).  A 16-bit
// logit is widened exactly on load; a gradient is rounded to nearest-even once, on store.  For X == T both are no-ops.
__device__ __forceinline__ float  widen(float x)         { return x; }
__device__ __forceinline__ double widen(double x)        { return x; }
__device__ __forceinline__ float  widen(__half x)        { return __half2float(x); }
__device__ __forceinline__ float  widen(__nv_bfloat16 x) { return __bfloat162float(x); }
template <typename X, typename T> __device__ __forceinline__ X narrow(T v) { return v; }
template <> __device__ __forceinline__ __half narrow<__half, float>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 narrow<__nv_bfloat16, float>(float v) { return __float2bfloat16_rn(v); }

// 16 bytes of logits as the vectorised kernels move them: 4 fp32 or 8 fp16 / bf16 elements, widened to fp32 in registers.
template <typename X> struct Vec16;
template <> struct Vec16<float> {
    static constexpr int N = 4, LOG2N = 2;
    using Raw = float4;
    __device__ static Raw neg_inf() { return make_float4(-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F); }
    __device__ static void widen(const Raw& r, float (&f)[N]) { f[0] = r.x; f[1] = r.y; f[2] = r.z; f[3] = r.w; }
    __device__ static Raw narrow(const float (&f)[N]) { return make_float4(f[0], f[1], f[2], f[3]); }
};
template <typename H2, typename X> struct Vec16Half {
    static constexpr int N = 8, LOG2N = 3;
    using Raw = uint4;
    __device__ static void widen(const Raw& r, float (&f)[N]) {
        const H2* h = reinterpret_cast<const H2*>(&r);
#pragma unroll
        for (int i = 0; i < 4; ++i) { f[2 * i] = rb::widen(h[i].x); f[2 * i + 1] = rb::widen(h[i].y); }
    }
    __device__ static Raw narrow(const float (&f)[N]) {
        Raw r;
        X* h = reinterpret_cast<X*>(&r);
#pragma unroll
        for (int i = 0; i < N; ++i) h[i] = rb::narrow<X, float>(f[i]);
        return r;
    }
};
template <> struct Vec16<__half> : Vec16Half<__half2, __half> {
    __device__ static Raw neg_inf() { return make_uint4(0xfc00fc00u, 0xfc00fc00u, 0xfc00fc00u, 0xfc00fc00u); }
};
template <> struct Vec16<__nv_bfloat16> : Vec16Half<__nv_bfloat162, __nv_bfloat16> {
    __device__ static Raw neg_inf() { return make_uint4(0xff80ff80u, 0xff80ff80u, 0xff80ff80u, 0xff80ff80u); }
};

// max of N values as a pairwise tree, and sum_i exp(f_i - m) added left to right (for N = 4 exactly the fp32 kernels'
// fmaxf(fmaxf(x, y), fmaxf(z, w)) and expf(x - m) + expf(y - m) + expf(z - m) + expf(w - m))
template <int N>
__device__ __forceinline__ float tree_max(const float* f) {
    if constexpr (N == 1) return f[0];
    else return fmaxf(tree_max<N / 2>(f), tree_max<N / 2>(f + N / 2));
}
template <int N>
__device__ __forceinline__ float sum_exp(const float (&f)[N], float m) {
    float t = expf(f[0] - m);
#pragma unroll
    for (int i = 1; i < N; ++i) t += expf(f[i] - m);
    return t;
}

template <typename T>
__device__ __forceinline__ T warp_max(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { T w = __shfl_xor_sync(0xffffffffu, v, o); v = w > v ? w : v; }
    return v;
}
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// FastEmit (Yu et al. 2021): the share of a cell's occupancy that leaves through its label arc,
//   rho = exp(lp_label(t,u) + beta(t,u+1) - beta(t,u)) in [0, 1],
// clamped to 1 so that rounding cannot push it above, and so that a cell with beta(t,u) = -inf (rho NaN or +inf; its
// occupancy is 0) gets a finite factor 1 + lambda*rho.
template <typename T>
__device__ __forceinline__ T fastemit_rho(T lp_label, T beta_next_u, T beta) {
    const T r = xexp(lp_label + beta_next_u - beta);
    return r < T(1) ? r : T(1);
}

// Alignment-restricted loss: per utterance b and lattice column u an inclusive frame window [lo[b*maxU+u], hi[b*maxU+u]]
// (int32, row stride maxU, entries at u >= U_b ignored).  Cell (t,u) is ALLOWED iff lo <= t <= hi (and t < T_b); both arcs
// leaving a cell that is not allowed have log-probability -inf.  Nothing is clamped: an empty or out-of-range window is an
// empty column.  lo == NULL: no restriction (every cell of the lattice is allowed).
struct Windows {
    const int* lo; const int* hi;
    __device__ __forceinline__ bool allows(int b, int t, int u, int maxU) const {
        if (!lo) return true;
        const long long k = (long long)b * maxU + u;
        return t >= lo[k] && t <= hi[k];
    }
};

struct CellIdx { int b, t, u; };
__device__ __forceinline__ CellIdx decode_cell(long long cell, int maxT, int maxU) {
    CellIdx c;
    c.u = (int)(cell % maxU);
    long long bt = cell / maxU;
    c.t = (int)(bt % maxT);
    c.b = (int)(bt / maxT);
    return c;
}
__device__ __forceinline__ long long sk_index(int b, int t, int u, int maxU, long long SK) {
    return (long long)b * SK + (long long)(t + u) * maxU + u;
}

// Prologue of the one-warp-per-row kernels (lse_gather, rnnt_grad): the warp's row of the chunk, and its lattice cell
// (natural cell row0 + row) with the utterance's extent.  A padded cell (t >= T_b or u >= U_b) is never read downstream.
__device__ __forceinline__ long long warp_row() { return ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
struct RowCell {
    long long cell;
    int b, t, u, Tn, Un;
    __device__ bool padded() const { return t >= Tn || u >= Un; }
    // padded, or outside the column's window: the cell is never read downstream and its gradient row is 0
    __device__ bool skipped(const Windows& w, int maxU) const { return padded() || !w.allows(b, t, u, maxU); }
    __device__ long long sk(int maxU, long long SK) const { return sk_index(b, t, u, maxU, SK); }
    // labels[b][u], -1 on the last column (no label arc)
    __device__ int label(const int* labels, int maxU) const { return u < Un - 1 ? labels[(long long)b * (maxU - 1) + u] : -1; }
};
__device__ __forceinline__ RowCell row_cell(long long cell, int maxT, int maxU, const int* xlen, const int* ylen) {
    const CellIdx c = decode_cell(cell, maxT, maxU);
    return {cell, c.b, c.t, c.u, xlen[c.b], ylen[c.b] + 1};
}

// Windows that admit no path leave ll = -inf: the utterance's cost is +inf and its gradients are exactly 0 (alpha + beta
// - ll is never formed for it).  Without windows ll is used as it comes.
template <typename T>
__device__ __forceinline__ bool win_infeasible(const Windows& w, T ll) { return w.lo && ll == neg_inf<T>(); }

// lane 0 of lse_gather: the row's log-softmax denominator (natural order) and its blank / label log-probs (skewed)
template <typename T, typename X>
__device__ __forceinline__ void store_lse_logprobs(const RowCell& c, const X* x, T l, int blank, const int* labels,
                                                   int maxU, long long SK, T* lse, T* lpb, T* lpl) {
    lse[c.cell] = l;
    const long long k = c.sk(maxU, SK);
    lpb[k] = widen(x[blank]) - l;
    if (c.u < c.Un - 1) lpl[k] = widen(x[c.label(labels, maxU)]) - l;
}

// Outgoing-arc terms of a valid cell (t,u), gpu_rnnt_kernel.h:163-172; beta points at beta(t,u) in the skewed plane, so
// beta(t+1,u) = beta[maxU] and beta(t,u+1) = beta[maxU + 1] (next diagonal), each read only where its arc exists:
//   sb = exp(alpha + lp_blank - ll (+ beta(t+1,u)))    (the last cell's blank arc leaves the lattice: no beta)
//   sl = exp(alpha + lp_label - ll + beta(t,u+1)),     times (1 + lambda) under FastEmit
// FastEmit (fe: lambda != 0 and a label arc) also gives lrho = lambda * fastemit_rho (else 0).  Callers combine the
// terms themselves: their bits depend on the exact expressions.
template <typename T>
struct ArcTerms { T sb, sl, lrho; bool fe; };
template <typename T>
__device__ __forceinline__ ArcTerms<T> arc_terms(T a, T ll, T lp_blank, T lp_label, const T* beta, int maxU, bool last,
                                                 bool t_inner, bool has_label, float fastemit_lambda) {
    ArcTerms<T> r{T(0), T(0), T(0), false};
    if (last) r.sb = xexp(a + lp_blank - ll);
    if (t_inner) r.sb = xexp(a + lp_blank - ll + beta[maxU]);
    if (has_label) r.sl = xexp(a + lp_label - ll + beta[maxU + 1]);
    if (fastemit_lambda != 0.f && has_label) {
        const T lam = fastemit_lambda;
        r.lrho = lam * fastemit_rho<T>(lp_label, beta[maxU + 1], beta[0]);
        r.sl *= T(1) + lam;
        r.fe = true;
    }
    return r;
}

// ---------------------------------------------------------------------------------------------
// lse + gather: one warp per lattice cell (row of V logits).  Row r of `logits` is natural cell
// row0 + r.  Two in-cache passes (max, then sum exp(x-max)) reproduce the reference's
// reduce_max / reduce_exp arithmetic; the row (<= 16 KB) is served by L1 on the second pass.
// Writes lse[cell] (natural order) and lp_blank / lp_label at the skewed index.  X: element type of the logits (T, or
// fp16 / bf16 over a float workspace).
// ---------------------------------------------------------------------------------------------
template <typename T, typename X = T>
__global__ void __launch_bounds__(256) lse_gather_kernel(const X* __restrict__ logits, long long row0,
                                                         long long nrows, int V, const int* __restrict__ xlen,
                                                         const int* __restrict__ ylen,
                                                         const int* __restrict__ labels, int maxT, int maxU,
                                                         long long SK, int blank, T* __restrict__ lse,
                                                         T* __restrict__ lpb, T* __restrict__ lpl, const Windows win) {
    const long long row = warp_row();
    const int lane = threadIdx.x & 31;
    if (row >= nrows) return;
    const RowCell c = row_cell(row0 + row, maxT, maxU, xlen, ylen);
    if (c.skipped(win, maxU)) return;
    const X* x = logits + row * (long long)V;
    T m = neg_inf<T>();
    for (int v = lane; v < V; v += 32) { T xv = widen(x[v]); m = xv > m ? xv : m; }
    m = warp_max(m);
    T s = 0;
    for (int v = lane; v < V; v += 32) s += xexp(widen(x[v]) - m);
    s = warp_sum(s);
    if (lane == 0) store_lse_logprobs(c, x, m + xlog(s), blank, labels, maxU, SK, lse, lpb, lpl);
}

// 16-byte fast path of lse_gather (V a multiple of Vec16<X>::N, 16-byte aligned rows): each lane streams 16-byte pieces
// of the row; rows of up to MAXV * 32 pieces (fp32: 1024 logits, fp16 / bf16: 2048) are held in registers between the
// max and the sum pass (ONE read of the logits), longer rows take the second pass from L1/L2.
template <typename X, int MAXV>   // per-lane 16-byte pieces held in registers (8); 0 -> always two passes
__global__ void __launch_bounds__(256) lse_gather_vec_kernel(const X* __restrict__ logits, long long row0,
                                                             long long nrows, int V, const int* __restrict__ xlen,
                                                             const int* __restrict__ ylen,
                                                             const int* __restrict__ labels, int maxT, int maxU,
                                                             long long SK, int blank, float* __restrict__ lse,
                                                             float* __restrict__ lpb, float* __restrict__ lpl,
                                                             const Windows win) {
    using P = Vec16<X>;
    const long long row = warp_row();
    const int lane = threadIdx.x & 31;
    if (row >= nrows) return;
    const RowCell c = row_cell(row0 + row, maxT, maxU, xlen, ylen);
    if (c.skipped(win, maxU)) return;
    const X* x = logits + row * (long long)V;
    const typename P::Raw* xv = reinterpret_cast<const typename P::Raw*>(x);
    const int nv = V >> P::LOG2N;
    float m = -CUDART_INF_F, s = 0.f;
    if (MAXV > 0 && nv <= MAXV * 32) {
        typename P::Raw r[MAXV > 0 ? MAXV : 1];
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int k = lane + 32 * i;
            r[i] = (k < nv) ? __ldg(xv + k) : P::neg_inf();
            float f[P::N];
            P::widen(r[i], f);
            m = fmaxf(m, tree_max<P::N>(f));
        }
        m = warp_max(m);
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            float f[P::N];
            P::widen(r[i], f);
            s += sum_exp(f, m);
        }
    } else {
        for (int k = lane; k < nv; k += 32) {
            float f[P::N];
            P::widen(__ldg(xv + k), f);
            m = fmaxf(m, tree_max<P::N>(f));
        }
        m = warp_max(m);
        for (int k = lane; k < nv; k += 32) {
            float f[P::N];
            P::widen(__ldg(xv + k), f);
            s += sum_exp(f, m);
        }
    }
    s = warp_sum(s);
    if (lane == 0) store_lse_logprobs(c, x, m + logf(s), blank, labels, maxU, SK, lse, lpb, lpl);
}

// 16-byte fast path of rnnt_grad_kernel (same arithmetic, 16-byte loads/stores; fp16 / bf16 gradients are rounded once,
// after the upstream gradient is multiplied in).
template <typename X>
__global__ void __launch_bounds__(256) rnnt_grad_vec_kernel(const X* logits, X* out, long long row0,
                                                            long long nrows, int V, const int* __restrict__ xlen,
                                                            const int* __restrict__ ylen,
                                                            const int* __restrict__ labels, int maxT, int maxU,
                                                            long long SK, int blank, const float* __restrict__ lse,
                                                            const float* __restrict__ alphas,
                                                            const float* __restrict__ betas,
                                                            const float* __restrict__ llf,
                                                            const float* __restrict__ gscale, float fastemit_lambda,
                                                            const Windows win) {
    using P = Vec16<X>;
    const long long row = warp_row();
    const int lane = threadIdx.x & 31;
    if (row >= nrows) return;
    const RowCell c = row_cell(row0 + row, maxT, maxU, xlen, ylen);
    const X* x = logits + row * (long long)V;
    const typename P::Raw* xv = reinterpret_cast<const typename P::Raw*>(x);
    typename P::Raw* gv = reinterpret_cast<typename P::Raw*>(out + row * (long long)V);
    const int nv = V >> P::LOG2N;
    if (c.skipped(win, maxU) || win_infeasible(win, llf[c.b])) {
        const float z[P::N] = {};
        for (int k = lane; k < nv; k += 32) gv[k] = P::narrow(z);
        return;
    }
    const long long k0 = c.sk(maxU, SK);
    const float a = alphas[k0], bt = betas[k0], ll = llf[c.b], l = lse[c.cell];
    const float gs = gscale ? gscale[c.b] : 1.f;
    const int label = c.label(labels, maxU);
    const bool last = c.t == c.Tn - 1 && c.u == c.Un - 1, t_inner = c.t < c.Tn - 1;
    const ArcTerms<float> arc = arc_terms<float>(a, ll, last || t_inner ? widen(x[blank]) - l : 0.f,
                                                 label >= 0 ? widen(x[label]) - l : 0.f, betas + k0, maxU, last, t_inner,
                                                 label >= 0, fastemit_lambda);
    float kd = a + bt - ll - l;
    if (arc.fe) kd += log1pf(arc.lrho);               // FastEmit: see rnnt_grad_kernel
    for (int k = lane; k < nv; k += 32) {
        float v[P::N], g[P::N];
        P::widen(xv[k], v);
#pragma unroll
        for (int i = 0; i < P::N; ++i) g[i] = expf(v[i] + kd);
        const int db = blank - (k << P::LOG2N), dl = label - (k << P::LOG2N);
#pragma unroll
        for (int i = 0; i < P::N; ++i) g[i] -= (db == i ? arc.sb : 0.f) + (dl == i ? arc.sl : 0.f);
#pragma unroll
        for (int i = 0; i < P::N; ++i) g[i] *= gs;
        gv[k] = P::narrow(g);
    }
}

// ---------------------------------------------------------------------------------------------
// alpha / beta wavefronts.  grid = (B, 2): blockIdx.y == 0 runs alpha, 1 runs beta, so the two
// recurrences of one utterance overlap on different SMs.  Thread u owns lattice column u and
// walks the anti-diagonals n = t+u; its own previous value stays in a register, the neighbour's
// arrives by warp shuffle; across warp boundaries through a shared-memory ring, with the warps running skewed
// by PF steps so that ONE __syncthreads per PF steps suffices (none when maxU <= 32).  The two cached log-probs of the thread's OWN
// cell are the only global reads: row n of the skewed planes, fully coalesced, software-prefetched
// PF rows ahead because they do not depend on the recurrence.
//   alpha(t,u) = LSE(alpha(t-1,u)+lpb(t-1,u), alpha(t,u-1)+lpl(t,u-1))        cpu_rnnt.h:182-195
//   beta(t,u)  = LSE(beta(t+1,u)+lpb(t,u),    beta(t,u+1)+lpl(t,u))            cpu_rnnt.h:223-236
//   llForward  = alpha(T-1,U-1)+lpb(T-1,U-1); llBackward = beta(0,0)           cpu_rnnt.h:209,251
// VIT (forward direction only) runs the same walk in the max-plus semiring: the Viterbi recurrence of forced alignment,
//   delta(t,u) = max(delta(t-1,u)+lpb(t-1,u), delta(t,u-1)+lpl(t,u-1)),   ll = delta(T-1,U-1)+lpb(T-1,U-1),
// with delta kept in registers only (`out` is not written).  Each warp records its decisions of a diagonal as ONE 32-bit
// ballot word, bit (u & 31) set when the label arc is STRICTLY greater (a tie goes to the blank arc):
//   dec[b*SKW + n*decw + (u >> 5)],  SKW = (maxT+maxU-1)*decw,  decw = ceil(maxU / 32).
// ---------------------------------------------------------------------------------------------
// WIN (alignment-restricted loss, struct Windows): thread u holds its column's window in two registers and a cell outside
// it FETCHES both log-probs as -inf, which is off the dependent chain; the recurrences themselves are unchanged.  The
// planes of cells outside the windows are never read, so nothing has to fill them.
template <typename T, int PF, bool BETA, bool VIT = false, bool WIN = false>
__device__ __forceinline__ void alpha_beta_body(const T* __restrict__ lpb, const T* __restrict__ lpl, T* __restrict__ out,
                                                T* __restrict__ ll, const int* __restrict__ xlen,
                                                const int* __restrict__ ylen, int maxU, long long SK,
                                                unsigned* __restrict__ dec = nullptr, int decw = 0,
                                                const Windows win = Windows{nullptr, nullptr}) {
    static_assert(!(VIT && BETA), "the Viterbi walk runs forward");
    const int b = blockIdx.x;
    const int u = threadIdx.x, lane = u & 31, warp = u >> 5;
    const int Tn = xlen[b], Un = ylen[b] + 1;
    const int nsteps = Tn + Un - 1;
    const int nwarps_blk = (int)(blockDim.x >> 5);
    const int nwarps = min(nwarps_blk, (Un + 31) >> 5);       // warps that own a column of THIS utterance
    const bool multi = nwarps_blk > 1;
    const bool col_ok = u < Un;
    // Cross-warp hand-over WITHOUT a barrier per step: the warps run SKEWED by PF steps -- warp w (alpha; mirrored for beta)
    // executes step i during macro iteration i / PF + w -- so everything a warp needs from its neighbour during a macro
    // iteration (the neighbour's edge-lane value of the PREVIOUS step, for each of its PF steps) was produced at least one
    // macro iteration earlier.  One __syncthreads per PF steps instead of one per step; the pipeline fill costs
    // (nwarps - 1) * PF extra steps.  Within a warp the anti-diagonal dependency is a shuffle.  The step itself is kept
    // free of branches, divisions and 64-bit multiplies: ONE warp per scheduler runs a chain of T+U-1 dependent steps, so
    // every instruction on it is latency (measured before: ~100 instructions and a dozen branches per step, 270 ns).
    constexpr int RING = 4 * PF;                      // edge values of the last 4 macro iterations per warp (power of two)
    static_assert((RING & (RING - 1)) == 0, "ring index is masked");
    __shared__ T mailbox[32][RING];

    const long long base = (long long)b * SK + u;
    const T NEG = neg_inf<T>();
    T own = NEG;     // alpha: alpha(t-1,u)+lpb(t-1,u)   beta: beta(t+1,u)
    T pass = NEG;    // alpha: alpha(t,u)+lpl(t,u)       beta: beta(t,u)   (handed to the neighbour)
    T result = 0;

    const int lag = (multi && warp < nwarps) ? (BETA ? nwarps - 1 - warp : warp) * PF : 0;   // this warp runs `lag` steps behind the first one
    const int src = BETA ? warp + 1 : warp - 1;                                  // neighbour warp whose edge lane feeds this one
    // (warps beyond the utterance's last column own nothing, run un-skewed and must not touch the ring: their reads would
    //  race with the working warps' writes of the same macro iteration)
    const bool has_src = BETA ? (warp + 1 < nwarps) : (warp > 0 && warp < nwarps);
    const bool edge_in = lane == (BETA ? 31 : 0), edge_out = multi && lane == (BETA ? 0 : 31);
    const int nmacro = (nsteps + PF - 1) / PF + (multi ? nwarps - 1 : 0);
    // step i works on diagonal n = i (alpha) / nsteps - 1 - i (beta): row n of the skewed planes, one pointer bump per step
    const long long dstep = BETA ? -(long long)maxU : (long long)maxU;
    // VIT: this warp's decision word of diagonal 0, one row of decw words per diagonal
    unsigned* pdec = VIT ? dec + (long long)b * (long long)(SK / maxU) * decw + warp : nullptr;
    T cb[PF], cl[PF], nb[PF], nl[PF];
    int wlo = 0, whi = -1;                            // WIN: this column's window
    if (WIN && col_ok) { wlo = win.lo[(long long)b * maxU + u]; whi = win.hi[(long long)b * maxU + u]; }
    auto fetch = [&](int i0, T* vb, T* vl) {
#pragma unroll
        for (int j = 0; j < PF; ++j) {
            const int i = i0 + j;
            const bool ok = col_ok && i >= 0 && i < nsteps;
            const long long off = base + (long long)(ok ? (BETA ? nsteps - 1 - i : i) : 0) * maxU;
            if constexpr (WIN) {
                const int t = (BETA ? nsteps - 1 - i : i) - u;
                const bool in = ok && t >= wlo && t <= whi;
                vb[j] = in ? lpb[off] : (ok ? NEG : T(0));
                vl[j] = in ? lpl[off] : (ok ? NEG : T(0));
            } else {
                vb[j] = ok ? lpb[off] : T(0);
                vl[j] = ok ? lpl[off] : T(0);
            }
        }
    };
    fetch(-lag, nb, nl);
    for (int m = 0; m < nmacro; ++m) {
        const int i0 = m * PF - lag;
#pragma unroll
        for (int j = 0; j < PF; ++j) { cb[j] = nb[j]; cl[j] = nl[j]; }
        fetch(i0 + PF, nb, nl);
        T* po = out + base + (long long)(BETA ? nsteps - 1 - i0 : i0) * maxU;     // row of step i0 (dereferenced only when in range)
        int t = (BETA ? nsteps - 1 - i0 : i0) - u;                                 // time index of this thread's cell at step i0
#pragma unroll
        for (int j = 0; j < PF; ++j, po += dstep, t += BETA ? -1 : 1) {
            const int i = i0 + j;
            if (i >= 0 && i < nsteps) {  // uniform across the warp
                T nbr = BETA ? __shfl_down_sync(0xffffffffu, pass, 1) : __shfl_up_sync(0xffffffffu, pass, 1);
                if (edge_in)      // the neighbour warp's edge value of step i - 1 (nothing before step 0)
                    nbr = (has_src && i > 0) ? mailbox[src][(i - 1) & (RING - 1)] : NEG;
                const bool active = col_ok && t >= 0 && t < Tn;
                const T vb = cb[j], vl = cl[j];
                T val;
                if (VIT) {
                    // delta(t,u) and its decision: the label arc wins only when strictly greater
                    const T emit = (u > 0) ? nbr : NEG;
                    const bool lab = emit > own;
                    val = (i == 0) ? T(0) : (lab ? emit : own);
                    const unsigned word = __ballot_sync(0xffffffffu, lab);
                    if (lane == 0 && warp < nwarps) pdec[(long long)i * decw] = word;
                } else if (!BETA) {
                    // alpha(t,u); own == -inf when t == 0, nbr is unused (forced -inf) when u == 0
                    const T emit = (u > 0) ? nbr : NEG;
                    val = (i == 0) ? T(0) : wave_lse(emit, own);
                } else {
                    const T no_emit = (t < Tn - 1) ? own + vb : NEG;
                    const T emit = (u < Un - 1) ? nbr + vl : NEG;
                    val = (t == Tn - 1 && u == Un - 1) ? vb : wave_lse(emit, no_emit);
                }
                if (active) {
                    if (!VIT) *po = val;
                    own = BETA ? val : val + vb;
                    pass = BETA ? val : val + vl;
                    result = own;      // alpha, last cell: alpha(T-1,U-1)+lpb(T-1,U-1);  beta, cell (0,0): beta(0,0)
                }
                if (edge_out && warp < nwarps) mailbox[warp][i & (RING - 1)] = pass;
            }
        }
        if (multi) __syncthreads();
    }
    if (!BETA && u == Un - 1) ll[b] = result;
    if (BETA && u == 0) ll[b] = result;
}

template <typename T, int PF>
__global__ void __launch_bounds__(1024) alpha_beta_kernel(const T* __restrict__ lpb, const T* __restrict__ lpl,
                                                          T* __restrict__ alphas, T* __restrict__ betas,
                                                          T* __restrict__ llf, T* __restrict__ llb,
                                                          const int* __restrict__ xlen,
                                                          const int* __restrict__ ylen, int maxU, long long SK) {
    if (blockIdx.y == 1) alpha_beta_body<T, PF, true>(lpb, lpl, betas, llb, xlen, ylen, maxU, SK);
    else alpha_beta_body<T, PF, false>(lpb, lpl, alphas, llf, xlen, ylen, maxU, SK);
}

// alpha_beta_kernel of the alignment-restricted loss (fp32): the same walk with the windows applied where the log-probs are
// fetched.  A kernel of its own, so that the unrestricted kernels keep their code.
template <int PF>
__global__ void __launch_bounds__(1024) alpha_beta_windowed_kernel(const float* __restrict__ lpb, const float* __restrict__ lpl,
                                                                   float* __restrict__ alphas, float* __restrict__ betas,
                                                                   float* __restrict__ llf, float* __restrict__ llb,
                                                                   const int* __restrict__ xlen, const int* __restrict__ ylen,
                                                                   int maxU, long long SK, const Windows win) {
    if (blockIdx.y == 1) alpha_beta_body<float, PF, true, false, true>(lpb, lpl, betas, llb, xlen, ylen, maxU, SK, nullptr, 0, win);
    else alpha_beta_body<float, PF, false, false, true>(lpb, lpl, alphas, llf, xlen, ylen, maxU, SK, nullptr, 0, win);
}

// Forced alignment, step 1: the Viterbi wavefront (alpha_beta_body<VIT>), one CTA per utterance.  Writes the decision
// bit-plane `dec` and best[b] = delta(T-1,U-1)+lpb(T-1,U-1), the log-probability of the single best alignment.
template <int PF>
__global__ void __launch_bounds__(1024) viterbi_kernel(const float* __restrict__ lpb, const float* __restrict__ lpl,
                                                       unsigned* __restrict__ dec, float* __restrict__ best,
                                                       const int* __restrict__ xlen, const int* __restrict__ ylen,
                                                       int maxU, long long SK) {
    alpha_beta_body<float, PF, false, true>(lpb, lpl, nullptr, best, xlen, ylen, maxU, SK, dec, (maxU + 31) >> 5);
}

// Forced alignment, step 2: the backtrace, one CTA per utterance.  The walk from (T-1,U-1) to (0,0) moves down exactly
// one diagonal per step, so the decision rows it reads are known before it starts: they are streamed into shared memory
// in chunks of BT_WORDS words, warps 1.. loading chunk c+1 while lane 0 of warp 0 walks chunk c, and every step of the
// walk costs one shared-memory read instead of a dependent L2 round trip.  On the lattice's edges the only predecessor
// is taken (t == 0: the label arc, u == 0: the blank arc), whatever the bit says.
//   frames[b*(maxU-1) + j] = t of the label arc (t,j) -> (t,j+1) on the best path;  -1 for j >= U_b - 1.
// overflow (nullable): the tensor-core forward's broken valid_tile_bound word: best = NaN and every frame -1.
constexpr int BT_THREADS = 256, BT_WORDS = 4096;
__global__ void __launch_bounds__(BT_THREADS) backtrace_kernel(const unsigned* __restrict__ dec, const float* __restrict__ vbest,
                                                               const int* __restrict__ overflow, const int* __restrict__ xlen,
                                                               const int* __restrict__ ylen, int maxT, int maxU,
                                                               float* __restrict__ best_logp, int* __restrict__ frames) {
    __shared__ unsigned buf[2][BT_WORDS];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int Tn = xlen[b], Un = ylen[b] + 1;
    const int decw = (maxU + 31) >> 5, wn = (Un + 31) >> 5;      // words per diagonal: stored / used by this utterance
    const bool bad = overflow && *overflow;
    int* fr = frames + (long long)b * (maxU - 1);
    for (int j = (bad ? 0 : Un - 1) + tid; j < maxU - 1; j += BT_THREADS) fr[j] = -1;
    if (tid == 0) best_logp[b] = bad ? __int_as_float(0x7fc00000) : vbest[b];
    if (bad) return;
    const unsigned* db = dec + (long long)b * (maxT + maxU - 1) * decw;
    const int top = Tn + Un - 2;                 // the walk reads diagonals top, top-1, ..., 1
    const int rows = BT_WORDS / wn;              // diagonals per chunk
    const int nchunks = (top + rows - 1) / rows;
    // chunk c holds diagonals top - c*rows down to max(1, top - (c+1)*rows + 1), word k at row top - c*rows - k / wn
    auto load = [&](int c, unsigned* dst, int l0, int nl) {
        const int hi = top - c * rows, lo = max(1, hi - rows + 1), n = (hi - lo + 1) * wn;
        for (int k = tid - l0; k < n; k += nl) {
            const int r = k / wn;
            dst[k] = db[(long long)(hi - r) * decw + (k - r * wn)];
        }
    };
    if (nchunks > 0) load(0, buf[0], 0, BT_THREADS);
    __syncthreads();
    int t = Tn - 1, u = Un - 1;
    for (int c = 0; c < nchunks; ++c) {
        if (tid >= 32 && c + 1 < nchunks) load(c + 1, buf[(c + 1) & 1], 32, BT_THREADS - 32);
        if (tid == 0) {
            const unsigned* s = buf[c & 1];
            const int hi = top - c * rows, lo = max(1, hi - rows + 1);
            for (int n = hi; n >= lo; --n) {
                const unsigned w = s[(hi - n) * wn + (u >> 5)];
                if (u > 0 && (t == 0 || ((w >> (u & 31)) & 1u))) { --u; fr[u] = t; }
                else --t;
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------
// Gradient w.r.t. logits, one warp per cell row -- gpu_rnnt_kernel.h:143-179:
//   g[v] = exp(alpha+beta+lp_v-ll) - [v==blank & last cell] exp(alpha+lp_v-ll)
//          - [v==blank & t<T-1] exp(alpha+lp_v-ll+beta(t+1,u)) - [v==label_u & u<U-1] exp(alpha+lp_v-ll+beta(t,u+1))
// normalised by llForward (gpu_rnnt.h:198-200).  Padded cells are written 0 here (the reference
// memsets the whole tensor first, gpu_rnnt.h:109).  `out` may alias `logits` (in-place, used by the
// exact joint path).  gscale (nullable): per-utterance upstream gradient, pre-multiplied.  X: element type of the
// logits and gradients (T, or fp16 / bf16 over a float workspace: one rounding, after the multiply).
// FastEmit (fastemit_lambda > 0): the label arc's gradient is scaled by (1 + lambda), so the row becomes
//   g[v] = (gamma + lambda*gamma_L) p_v - [v==blank] gamma_B - [v==label_u] (1 + lambda) gamma_L,
// gamma_L = sl; the softmax term is today's times (1 + lambda*rho) (fastemit_rho), i.e. kd += log1p(lambda*rho).
// arc_terms forms sb, sl and lambda*rho; lambda == 0 takes none of the FastEmit arithmetic: the result is bit-identical
// to the plain loss.
// ---------------------------------------------------------------------------------------------
template <typename T, typename X = T>
__global__ void __launch_bounds__(256) rnnt_grad_kernel(const X* logits, X* out, long long row0, long long nrows,
                                                        int V, const int* __restrict__ xlen,
                                                        const int* __restrict__ ylen,
                                                        const int* __restrict__ labels, int maxT, int maxU,
                                                        long long SK, int blank, const T* __restrict__ lse,
                                                        const T* __restrict__ alphas, const T* __restrict__ betas,
                                                        const T* __restrict__ llf, const T* __restrict__ gscale,
                                                        float fastemit_lambda, const Windows win) {
    const long long row = warp_row();
    const int lane = threadIdx.x & 31;
    if (row >= nrows) return;
    const RowCell c = row_cell(row0 + row, maxT, maxU, xlen, ylen);
    const X* x = logits + row * (long long)V;
    X* g = out + row * (long long)V;
    if (c.skipped(win, maxU) || win_infeasible(win, llf[c.b])) {
        for (int v = lane; v < V; v += 32) g[v] = narrow<X>(T(0));
        return;
    }
    const long long k = c.sk(maxU, SK);
    const T a = alphas[k], bt = betas[k], ll = llf[c.b], l = lse[c.cell];
    const T gs = gscale ? gscale[c.b] : T(1);
    const int label = c.label(labels, maxU);
    const bool last = c.t == c.Tn - 1 && c.u == c.Un - 1, t_inner = c.t < c.Tn - 1;
    const ArcTerms<T> arc = arc_terms<T>(a, ll, last || t_inner ? widen(x[blank]) - l : T(0),
                                         label >= 0 ? widen(x[label]) - l : T(0), betas + k, maxU, last, t_inner,
                                         label >= 0, fastemit_lambda);
    T kd = a + bt - ll - l;
    if (arc.fe) kd += xlog1p(arc.lrho);
    for (int v = lane; v < V; v += 32) {
        T gr = xexp(widen(x[v]) + kd);
        if (v == blank) gr -= arc.sb;
        if (v == label) gr -= arc.sl;
        g[v] = narrow<X>(gr * gs);
    }
}

// Per-ROW scale of the tensor-core backward, in the row order of the kept arrays (row = slot*128 + r, r = tl*8 + ul of a
// 16 x 8 tile), and the patch of the row's two special columns:
//   dlogit[row, v] = g * exp(x_v + kd) = rs * E[row, v],   E = 2^(y_v - ref) kept by the forward (bf16),
//   rs = g * 2^(ref + kd2),  kd2 = (alpha + beta - ll - lse) * log2(e)                       (gpu_rnnt_kernel.h:143-161)
// except for v = blank and v = label_u, whose outgoing-arc terms (gpu_rnnt_kernel.h:163-172) are subtracted: their FINAL
// values dl_blank, dl_label are formed here from the cached log-probs and stored as E' = dl / rs in place of E, so that
// rs * E' is exact for them too.  Rows outside the valid lattice get rs = 0 (their E stays finite: it was formed from z = 0).
// FastEmit (fastemit_lambda > 0, see rnnt_grad_kernel): rs is multiplied by fe = 1 + lambda*rho and the label arc's term
// by 1 + lambda (both from arc_terms), which the patched columns absorb; lambda == 0 leaves fe = 1 and every value
// bit-identical.
__global__ void __launch_bounds__(256) row_scale_kernel(const int* __restrict__ tile_of_slot, const int* __restrict__ count, int b0,
                                                        int nTb, int nUb, const int* __restrict__ xlen, const int* __restrict__ ylen,
                                                        const int* __restrict__ labels, int blank, int maxT, int maxU, long long SK,
                                                        const float* __restrict__ lse, const float* __restrict__ lpb,
                                                        const float* __restrict__ lpl, const float* __restrict__ alphas,
                                                        const float* __restrict__ betas, const float* __restrict__ llf,
                                                        const float* __restrict__ gscale, const float* __restrict__ rowref, int V,
                                                        unsigned short* __restrict__ E, float* __restrict__ rowscale,
                                                        float fastemit_lambda, const Windows win) {
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int sl = (int)(row >> 7), r = (int)(row & 127);
    if (sl >= *count) return;
    const int tile = tile_of_slot[sl], per_utt = nTb * nUb;
    const int bl = tile / per_utt, rem = tile - bl * per_utt, b = b0 + bl;
    const int t = (rem / nUb) * 16 + (r >> 3), u = (rem % nUb) * 8 + (r & 7);
    const int Tn = xlen[b], Un = ylen[b] + 1;
    float rs = 0.f;
    // (rows outside their column's window, and every row of an utterance whose windows admit no path, keep rs = 0 and
    //  their E untouched: nothing of theirs reaches a gradient)
    if (t < Tn && u < Un && win.allows(b, t, u, maxU) && !win_infeasible(win, llf[b])) {
        const long long k = sk_index(b, t, u, maxU, SK);
        const float a = alphas[k], bt = betas[k], ll = llf[b], g = gscale ? gscale[b] : 1.f;
        const float occ = a + bt - ll;                                   // log occupancy of the cell
        const bool has_label = u < Un - 1;
        const float lp_label = has_label ? lpl[k] : 0.f;
        const ArcTerms<float> arc = arc_terms<float>(a, ll, lpb[k], lp_label, betas + k, maxU, t == Tn - 1 && u == Un - 1,
                                                     t < Tn - 1, has_label, fastemit_lambda);
        const float pl = has_label ? expf(lp_label + occ) : 0.f;
        const int lab = has_label ? labels[(long long)b * (maxU - 1) + u] : -1;
        const float fe = arc.fe ? 1.f + arc.lrho : 1.f;                  // FastEmit factor of the softmax term
        float dlb = g * (fe * expf(lpb[k] + occ) - arc.sb), dll = g * (fe * pl - arc.sl);
        if (has_label && lab == blank) { dlb -= g * arc.sl; dll = dlb; } // degenerate: label == blank
        rs = fe * (g * exp2f(rowref[row] + (occ - lse[((long long)b * maxT + t) * maxU + u]) * 1.4426950408889634f));
        // rs is cut to 0 only where 1/rs stops being finite (a denormal rs would make it +inf and the patched columns NaN).
        // The forward keeps lse2 - ref <= FWD_REBASE + log2 V, so a row cut here has |g| * e^occ < 2^-126 * 2^(64 + log2 V):
        // at V = 4096 below 2^-50, against rows of up to |g|.  The patched columns dl / rs are at most 2^(lse2 - ref),
        // i.e. 2^76 at V = 4096, whatever g is: far inside the bf16 range.
        // A cell of occupancy below 2^-64 whose rs is below 1e-30 is treated as 0 as well: its whole gradient row is below
        // 2^-64 |g|, far under the fp32 resolution of every sum it joins, and bwd_dz_kernel skips the epilogue of rows
        // with rs == 0.  (A cut on rs alone would also drop rows that matter once g or 2^(ref - lse2) is small.)
        const float ars = fabsf(rs);
        if (!(ars >= 1.17549435e-38f && ars < CUDART_INF_F) || (ars < 1e-30f && occ < -64.f * 0.6931471805599453f))
            rs = 0.f;                                                    // 1.17549435e-38 = FLT_MIN
        const float inv = rs != 0.f ? 1.f / rs : 0.f;
        unsigned short* e = E + row * (long long)V;
        e[blank] = __bfloat16_as_ushort(__float2bfloat16(dlb * inv));
        if (lab >= 0) e[lab] = __bfloat16_as_ushort(__float2bfloat16(dll * inv));
    }
    rowscale[row] = rs;
}

// ---------------------------------------------------------------------------------------------
// fp32 exact joint path building blocks
// ---------------------------------------------------------------------------------------------
// z[r,h] = tanh(enc[b,t,h] + pred[b,u,h]) for natural cells row0 .. row0+nrows   (model.py:158-163)
__global__ void __launch_bounds__(256) zgen_kernel(const float* __restrict__ enc, const float* __restrict__ pred,
                                                   float* __restrict__ z, long long row0, long long nrows, int maxT,
                                                   int maxU, int H) {
    const long long total = nrows * H;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / H;
        const int h = (int)(i - r * H);
        const CellIdx c = decode_cell(row0 + r, maxT, maxU);
        z[i] = tanhf(enc[((long long)c.b * maxT + c.t) * H + h] + pred[((long long)c.b * maxU + c.u) * H + h]);
    }
}

// C[m,n] = (accumulate ? C : 0) + sum_k A(m,k) B(k,n) (+ bias[n]); generic strides so that the three
// products of the exact path (Z.W, dL.W^T, Z^T.dL) share one kernel.  64x64x16 tiles, 256 threads,
// 4x4 register micro-tiles; the smem tile loads pick the thread mapping by which stride is unit.
template <bool A_K_CONTIG, bool B_N_CONTIG>
__global__ void __launch_bounds__(256) sgemm_kernel(const float* __restrict__ A, const float* __restrict__ Bm,
                                                    float* __restrict__ C, const float* __restrict__ bias, int M,
                                                    int N, int K, long long sAm, long long sAk, long long sBk,
                                                    long long sBn, long long ldc, int accumulate) {
    constexpr int BM = 64, BN = 64, BK = 16;
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[BK][BN + 4];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int tx = tid & 15, ty = tid >> 4;  // 16 x 16 threads, 4x4 outputs each
    float acc[4][4] = {};
    for (int k0 = 0; k0 < K; k0 += BK) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {  // 1024 elements per operand tile, 4 per thread
            const int e = tid + i * 256;
            int am, ak;
            if (A_K_CONTIG) { ak = e & 15; am = e >> 4; } else { am = e & 63; ak = e >> 6; }
            const int gm = m0 + am, gk = k0 + ak;
            As[ak][am] = (gm < M && gk < K) ? A[gm * sAm + gk * sAk] : 0.f;
            int bn, bk;
            if (B_N_CONTIG) { bn = e & 63; bk = e >> 6; } else { bk = e & 15; bn = e >> 4; }
            const int gn = n0 + bn, gk2 = k0 + bk;
            Bs[bk][bn] = (gn < N && gk2 < K) ? Bm[gk2 * sBk + gn * sBn] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = Bs[k][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int gm = m0 + ty * 4 + i;
        if (gm >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int gn = n0 + tx * 4 + j;
            if (gn >= N) continue;
            float v = acc[i][j] + (bias ? bias[gn] : 0.f);
            float* c = C + (long long)gm * ldc + gn;
            *c = accumulate ? *c + v : v;
        }
    }
}

// Faster fp32 GEMM for the exact path: 128x128x8 tiles, 256 threads, 8x8 register micro-tiles (as 2x2 blocks of
// 4x4 so that every smem read is a conflict-free float4), 16-byte global loads along whichever dimension is
// contiguous.  Requirements (checked by the launcher, else sgemm_kernel is used): the contiguous dimension of each
// operand is a multiple of 4 and 16-byte aligned.  Same semantics as sgemm_kernel.
template <bool A_K_CONTIG, bool B_N_CONTIG>
__global__ void __launch_bounds__(256) sgemm128_kernel(const float* __restrict__ A, const float* __restrict__ Bm,
                                                       float* __restrict__ C, const float* __restrict__ bias, int M,
                                                       int N, int K, long long sAm, long long sAk, long long sBk,
                                                       long long sBn, long long ldc, int accumulate) {
    constexpr int BM = 128, BN = 128, BK = 8;
    __shared__ __align__(16) float As[2][BK][BM];
    __shared__ __align__(16) float Bs[2][BK][BN];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int tx = tid & 15, ty = tid >> 4;
    // split-K: blockIdx.z owns K range [kbeg, kend); partial products are combined with atomicAdd (accumulate != 0)
    const int kchunk = ((K + (int)gridDim.z - 1) / (int)gridDim.z + BK - 1) / BK * BK;
    const int kbeg = blockIdx.z * kchunk, kend = min(K, kbeg + kchunk);
    if (kbeg >= kend) return;
    float acc[8][8] = {};
    float4 ra, rb;
    auto gload = [&](int k0) {
        if (A_K_CONTIG) {   // one float4 along k: row m = tid/2, k4 = (tid&1)*4
            const int m = m0 + (tid >> 1), k = k0 + (tid & 1) * 4;
            ra = (m < M && k < K) ? *reinterpret_cast<const float4*>(A + m * sAm + k) : make_float4(0.f, 0.f, 0.f, 0.f);
        } else {            // one float4 along m: k = tid/32, m4 = (tid&31)*4
            const int k = k0 + (tid >> 5), m = m0 + (tid & 31) * 4;
            ra = (m < M && k < K) ? *reinterpret_cast<const float4*>(A + k * sAk + m) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        if (B_N_CONTIG) {
            const int k = k0 + (tid >> 5), n = n0 + (tid & 31) * 4;
            rb = (n < N && k < K) ? *reinterpret_cast<const float4*>(Bm + k * sBk + n) : make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
            const int n = n0 + (tid >> 1), k = k0 + (tid & 1) * 4;
            rb = (n < N && k < K) ? *reinterpret_cast<const float4*>(Bm + n * sBn + k) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto sstore = [&](int buf) {
        if (A_K_CONTIG) {
            const int m = tid >> 1, k = (tid & 1) * 4;
            As[buf][k][m] = ra.x; As[buf][k + 1][m] = ra.y; As[buf][k + 2][m] = ra.z; As[buf][k + 3][m] = ra.w;
        } else {
            *reinterpret_cast<float4*>(&As[buf][tid >> 5][(tid & 31) * 4]) = ra;
        }
        if (B_N_CONTIG) {
            *reinterpret_cast<float4*>(&Bs[buf][tid >> 5][(tid & 31) * 4]) = rb;
        } else {
            const int n = tid >> 1, k = (tid & 1) * 4;
            Bs[buf][k][n] = rb.x; Bs[buf][k + 1][n] = rb.y; Bs[buf][k + 2][n] = rb.z; Bs[buf][k + 3][n] = rb.w;
        }
    };
    K = kend;                      // the guards in gload() compare against the end of this block's K range
    gload(kbeg);
    sstore(0);
    __syncthreads();
    int buf = 0;
    for (int k0 = kbeg; k0 < K; k0 += BK) {
        if (k0 + BK < K) gload(k0 + BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (k0 + BK < K) {
            sstore(buf ^ 1);
            __syncthreads();
            buf ^= 1;
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int gm = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
        if (gm >= M) continue;
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
            const int gn = n0 + jj * 64 + tx * 4;
            if (gn >= N) continue;   // N % 4 == 0: a float4 is either fully inside or fully outside
            float4 v = make_float4(acc[i][jj * 4], acc[i][jj * 4 + 1], acc[i][jj * 4 + 2], acc[i][jj * 4 + 3]);
            if (bias && blockIdx.z == 0) { const float4 bb = *reinterpret_cast<const float4*>(bias + gn); v.x += bb.x; v.y += bb.y; v.z += bb.z; v.w += bb.w; }
            float* cp = C + (long long)gm * ldc + gn;
            if (gridDim.z > 1) {   // split-K: C was zero-initialised (or holds earlier chunks); bias added by split 0 only
                atomicAdd(cp, v.x); atomicAdd(cp + 1, v.y); atomicAdd(cp + 2, v.z); atomicAdd(cp + 3, v.w);
            } else {
                float4* c = reinterpret_cast<float4*>(cp);
                if (accumulate) { const float4 o = *c; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
                *c = v;
            }
        }
    }
}

// dpre = dz * (1 - z^2); d_enc[b,t,:] += sum_u dpre, d_pred[b,u,:] += sum_t dpre (atomics; exact path only)
__global__ void __launch_bounds__(256) dz_reduce_kernel(const float* __restrict__ dz, const float* __restrict__ z,
                                                        long long row0, long long nrows, int maxT, int maxU, int H,
                                                        float* __restrict__ d_enc, float* __restrict__ d_pred) {
    const long long total = nrows * H;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / H;
        const int h = (int)(i - r * H);
        const CellIdx c = decode_cell(row0 + r, maxT, maxU);
        const float zz = z[i];
        const float g = dz[i] * (1.f - zz * zz);
        if (g != 0.f) {
            atomicAdd(d_enc + ((long long)c.b * maxT + c.t) * H + h, g);
            atomicAdd(d_pred + ((long long)c.b * maxU + c.u) * H + h, g);
        }
    }
}

// out[v] += sum_r x[r,v]   (db of the exact path, db1 of dense1): one block per 32 columns and gridDim.y row blocks of 8
// row lanes.  With gridDim.y == 1 each column has one writer and a fixed summation order: run-to-run deterministic.
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, long long nrows, int V,
                                                     float* __restrict__ out) {
    const int v = blockIdx.x * 32 + (threadIdx.x & 31);
    const int ry = threadIdx.x >> 5;  // 8 row lanes
    float s = 0.f;
    if (v < V)
        for (long long r = blockIdx.y * 8 + ry; r < nrows; r += (long long)gridDim.y * 8) s += x[r * V + v];
    __shared__ float sm[8][33];
    sm[ry][threadIdx.x & 31] = s;
    __syncthreads();
    if (ry == 0 && v < V) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x & 31];
        atomicAdd(out + v, t);
    }
}

}  // namespace rb
