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
//   row_scale_kernel    per-row scales of the tensor-core backward GEMMs + the patch of the two special columns
//   zgen/sgemm/...      fp32 building blocks of the exact (RNNTB200_FP32_EXACT) joint path
//
// Data layout ("skewed" planes): a per-utterance plane stores cell (t,u) at row n=t+u, column u:
//     sk(b,t,u) = b*SK + (t+u)*maxU + u,   SK = (maxT+maxU-1)*maxU
// so that step n of a wavefront touches ONE contiguous row (coalesced), which the reference's
// (t*maxU+u) planes cannot offer (stride maxU-1 between neighbouring threads).
#pragma once
#include <cuda_bf16.h>
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

// ---------------------------------------------------------------------------------------------
// lse + gather: one warp per lattice cell (row of V logits).  Row r of `logits` is natural cell
// row0 + r.  Two in-cache passes (max, then sum exp(x-max)) reproduce the reference's
// reduce_max / reduce_exp arithmetic; the row (<= 16 KB) is served by L1 on the second pass.
// Writes lse[cell] (natural order) and lp_blank / lp_label at the skewed index.
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) lse_gather_kernel(const T* __restrict__ logits, long long row0,
                                                         long long nrows, int V, const int* __restrict__ xlen,
                                                         const int* __restrict__ ylen,
                                                         const int* __restrict__ labels, int maxT, int maxU,
                                                         long long SK, int blank, T* __restrict__ lse,
                                                         T* __restrict__ lpb, T* __restrict__ lpl) {
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= nrows) return;
    const long long cell = row0 + row;
    const CellIdx c = decode_cell(cell, maxT, maxU);
    const int Tn = xlen[c.b], Un = ylen[c.b] + 1;
    if (c.t >= Tn || c.u >= Un) return;  // padded cell: never read downstream
    const T* x = logits + row * (long long)V;
    T m = neg_inf<T>();
    for (int v = lane; v < V; v += 32) { T xv = x[v]; m = xv > m ? xv : m; }
    m = warp_max(m);
    T s = 0;
    for (int v = lane; v < V; v += 32) s += xexp(x[v] - m);
    s = warp_sum(s);
    if (lane == 0) {
        const T l = m + xlog(s);
        lse[cell] = l;
        const long long k = sk_index(c.b, c.t, c.u, maxU, SK);
        lpb[k] = x[blank] - l;
        if (c.u < Un - 1) lpl[k] = x[labels[(long long)c.b * (maxU - 1) + c.u]] - l;
    }
}

// float4 fast path of lse_gather (V % 4 == 0, 16-byte aligned rows): each lane streams 16-byte pieces of the row;
// rows of up to 1024 logits are held in registers between the max and the sum pass (ONE read of the logits),
// longer rows take the second pass from L1/L2.
template <int MAXV4>   // per-lane float4 capacity held in registers (8 -> V <= 1024); 0 -> always two passes
__global__ void __launch_bounds__(256) lse_gather_vec_kernel(const float* __restrict__ logits, long long row0,
                                                             long long nrows, int V, const int* __restrict__ xlen,
                                                             const int* __restrict__ ylen,
                                                             const int* __restrict__ labels, int maxT, int maxU,
                                                             long long SK, int blank, float* __restrict__ lse,
                                                             float* __restrict__ lpb, float* __restrict__ lpl) {
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= nrows) return;
    const long long cell = row0 + row;
    const CellIdx c = decode_cell(cell, maxT, maxU);
    const int Tn = xlen[c.b], Un = ylen[c.b] + 1;
    if (c.t >= Tn || c.u >= Un) return;
    const float* x = logits + row * (long long)V;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    const int n4 = V >> 2;
    float m = -CUDART_INF_F, s = 0.f;
    if (MAXV4 > 0 && n4 <= MAXV4 * 32) {
        float4 r[MAXV4 > 0 ? MAXV4 : 1];
#pragma unroll
        for (int i = 0; i < MAXV4; ++i) {
            const int k = lane + 32 * i;
            r[i] = (k < n4) ? __ldg(x4 + k) : make_float4(-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F);
            m = fmaxf(m, fmaxf(fmaxf(r[i].x, r[i].y), fmaxf(r[i].z, r[i].w)));
        }
        m = warp_max(m);
#pragma unroll
        for (int i = 0; i < MAXV4; ++i) s += expf(r[i].x - m) + expf(r[i].y - m) + expf(r[i].z - m) + expf(r[i].w - m);
    } else {
        for (int k = lane; k < n4; k += 32) {
            const float4 v = __ldg(x4 + k);
            m = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
        }
        m = warp_max(m);
        for (int k = lane; k < n4; k += 32) {
            const float4 v = __ldg(x4 + k);
            s += expf(v.x - m) + expf(v.y - m) + expf(v.z - m) + expf(v.w - m);
        }
    }
    s = warp_sum(s);
    if (lane == 0) {
        const float l = m + logf(s);
        lse[cell] = l;
        const long long k = sk_index(c.b, c.t, c.u, maxU, SK);
        lpb[k] = x[blank] - l;
        if (c.u < Un - 1) lpl[k] = x[labels[(long long)c.b * (maxU - 1) + c.u]] - l;
    }
}

// float4 fast path of rnnt_grad_kernel (same arithmetic, 16-byte loads/stores).
__global__ void __launch_bounds__(256) rnnt_grad_vec_kernel(const float* logits, float* out, long long row0,
                                                            long long nrows, int V, const int* __restrict__ xlen,
                                                            const int* __restrict__ ylen,
                                                            const int* __restrict__ labels, int maxT, int maxU,
                                                            long long SK, int blank, const float* __restrict__ lse,
                                                            const float* __restrict__ alphas,
                                                            const float* __restrict__ betas,
                                                            const float* __restrict__ llf,
                                                            const float* __restrict__ gscale) {
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= nrows) return;
    const long long cell = row0 + row;
    const CellIdx c = decode_cell(cell, maxT, maxU);
    const int Tn = xlen[c.b], Un = ylen[c.b] + 1;
    const float* x = logits + row * (long long)V;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    float4* g4 = reinterpret_cast<float4*>(out + row * (long long)V);
    const int n4 = V >> 2;
    if (c.t >= Tn || c.u >= Un) {
        for (int k = lane; k < n4; k += 32) g4[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        return;
    }
    const long long k0 = sk_index(c.b, c.t, c.u, maxU, SK);
    const float a = alphas[k0], bt = betas[k0], ll = llf[c.b], l = lse[cell];
    const float gs = gscale ? gscale[c.b] : 1.f;
    const int label = (c.u < Un - 1) ? labels[(long long)c.b * (maxU - 1) + c.u] : -1;
    float sb = 0.f, sl = 0.f;
    if (c.t == Tn - 1 && c.u == Un - 1) sb = expf(a + (x[blank] - l) - ll);
    if (c.t < Tn - 1) sb = expf(a + (x[blank] - l) - ll + betas[k0 + maxU]);
    if (label >= 0) sl = expf(a + (x[label] - l) - ll + betas[k0 + maxU + 1]);
    const float kd = a + bt - ll - l;
    for (int k = lane; k < n4; k += 32) {
        const float4 v = x4[k];
        float4 g = make_float4(expf(v.x + kd), expf(v.y + kd), expf(v.z + kd), expf(v.w + kd));
        const int db = blank - (k << 2), dl = label - (k << 2);
        g.x -= (db == 0 ? sb : 0.f) + (dl == 0 ? sl : 0.f);
        g.y -= (db == 1 ? sb : 0.f) + (dl == 1 ? sl : 0.f);
        g.z -= (db == 2 ? sb : 0.f) + (dl == 2 ? sl : 0.f);
        g.w -= (db == 3 ? sb : 0.f) + (dl == 3 ? sl : 0.f);
        g.x *= gs; g.y *= gs; g.z *= gs; g.w *= gs;
        g4[k] = g;
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
// ---------------------------------------------------------------------------------------------
template <typename T, int PF, bool BETA>
__device__ __forceinline__ void alpha_beta_body(const T* __restrict__ lpb, const T* __restrict__ lpl, T* __restrict__ out,
                                                T* __restrict__ ll, const int* __restrict__ xlen,
                                                const int* __restrict__ ylen, int maxU, long long SK) {
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
    T cb[PF], cl[PF], nb[PF], nl[PF];
    auto fetch = [&](int i0, T* vb, T* vl) {
#pragma unroll
        for (int j = 0; j < PF; ++j) {
            const int i = i0 + j;
            const bool ok = col_ok && i >= 0 && i < nsteps;
            const long long off = base + (long long)(ok ? (BETA ? nsteps - 1 - i : i) : 0) * maxU;
            vb[j] = ok ? lpb[off] : T(0);
            vl[j] = ok ? lpl[off] : T(0);
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
                if (!BETA) {
                    // alpha(t,u); own == -inf when t == 0, nbr is unused (forced -inf) when u == 0
                    const T emit = (u > 0) ? nbr : NEG;
                    val = (i == 0) ? T(0) : wave_lse(emit, own);
                } else {
                    const T no_emit = (t < Tn - 1) ? own + vb : NEG;
                    const T emit = (u < Un - 1) ? nbr + vl : NEG;
                    val = (t == Tn - 1 && u == Un - 1) ? vb : wave_lse(emit, no_emit);
                }
                if (active) {
                    *po = val;
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

// ---------------------------------------------------------------------------------------------
// Gradient w.r.t. logits, one warp per cell row -- gpu_rnnt_kernel.h:143-179:
//   g[v] = exp(alpha+beta+lp_v-ll) - [v==blank & last cell] exp(alpha+lp_v-ll)
//          - [v==blank & t<T-1] exp(alpha+lp_v-ll+beta(t+1,u)) - [v==label_u & u<U-1] exp(alpha+lp_v-ll+beta(t,u+1))
// normalised by llForward (gpu_rnnt.h:198-200).  Padded cells are written 0 here (the reference
// memsets the whole tensor first, gpu_rnnt.h:109).  `out` may alias `logits` (in-place, used by the
// exact joint path).  gscale (nullable): per-utterance upstream gradient, pre-multiplied.
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) rnnt_grad_kernel(const T* logits, T* out, long long row0, long long nrows,
                                                        int V, const int* __restrict__ xlen,
                                                        const int* __restrict__ ylen,
                                                        const int* __restrict__ labels, int maxT, int maxU,
                                                        long long SK, int blank, const T* __restrict__ lse,
                                                        const T* __restrict__ alphas, const T* __restrict__ betas,
                                                        const T* __restrict__ llf, const T* __restrict__ gscale) {
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= nrows) return;
    const long long cell = row0 + row;
    const CellIdx c = decode_cell(cell, maxT, maxU);
    const int Tn = xlen[c.b], Un = ylen[c.b] + 1;
    const T* x = logits + row * (long long)V;
    T* g = out + row * (long long)V;
    if (c.t >= Tn || c.u >= Un) {
        for (int v = lane; v < V; v += 32) g[v] = T(0);
        return;
    }
    const long long k = sk_index(c.b, c.t, c.u, maxU, SK);
    const T a = alphas[k], bt = betas[k], ll = llf[c.b], l = lse[cell];
    const T gs = gscale ? gscale[c.b] : T(1);
    const int label = (c.u < Un - 1) ? labels[(long long)c.b * (maxU - 1) + c.u] : -1;
    T sb = 0, sl = 0;
    if (c.t == Tn - 1 && c.u == Un - 1) sb = xexp(a + (x[blank] - l) - ll);
    if (c.t < Tn - 1) sb = xexp(a + (x[blank] - l) - ll + betas[k + maxU]);        // beta(t+1,u): next diagonal, same column
    if (label >= 0) sl = xexp(a + (x[label] - l) - ll + betas[k + maxU + 1]);      // beta(t,u+1): next diagonal, next column
    const T kd = a + bt - ll - l;
    for (int v = lane; v < V; v += 32) {
        T gr = xexp(x[v] + kd);
        if (v == blank) gr -= sb;
        if (v == label) gr -= sl;
        g[v] = gr * gs;
    }
}

// Per-ROW scale of the tensor-core backward, in the row order of the kept arrays (row = slot*128 + r, r = tl*8 + ul of a
// 16 x 8 tile), and the patch of the row's two special columns:
//   dlogit[row, v] = g * exp(x_v + kd) = rs * E[row, v],   E = 2^(y_v - ref) kept by the forward (bf16),
//   rs = g * 2^(ref + kd2),  kd2 = (alpha + beta - ll - lse) * log2(e)                       (gpu_rnnt_kernel.h:143-161)
// except for v = blank and v = label_u, whose outgoing-arc terms (gpu_rnnt_kernel.h:163-172) are subtracted: their FINAL
// values dl_blank, dl_label are formed here from the cached log-probs and stored as E' = dl / rs in place of E, so that
// rs * E' is exact for them too.  Rows outside the valid lattice get rs = 0 (their E stays finite: it was formed from z = 0).
__global__ void __launch_bounds__(256) row_scale_kernel(const int* __restrict__ tile_of_slot, const int* __restrict__ count, int b0,
                                                        int nTb, int nUb, const int* __restrict__ xlen, const int* __restrict__ ylen,
                                                        const int* __restrict__ labels, int blank, int maxT, int maxU, long long SK,
                                                        const float* __restrict__ lse, const float* __restrict__ lpb,
                                                        const float* __restrict__ lpl, const float* __restrict__ alphas,
                                                        const float* __restrict__ betas, const float* __restrict__ llf,
                                                        const float* __restrict__ gscale, const float* __restrict__ rowref, int V,
                                                        unsigned short* __restrict__ E, float* __restrict__ rowscale) {
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int sl = (int)(row >> 7), r = (int)(row & 127);
    if (sl >= *count) return;
    const int tile = tile_of_slot[sl], per_utt = nTb * nUb;
    const int bl = tile / per_utt, rem = tile - bl * per_utt, b = b0 + bl;
    const int t = (rem / nUb) * 16 + (r >> 3), u = (rem % nUb) * 8 + (r & 7);
    const int Tn = xlen[b], Un = ylen[b] + 1;
    float rs = 0.f;
    if (t < Tn && u < Un) {
        const long long k = sk_index(b, t, u, maxU, SK);
        const float a = alphas[k], bt = betas[k], ll = llf[b], g = gscale ? gscale[b] : 1.f;
        const float occ = a + bt - ll;                                   // log occupancy of the cell
        float sb = 0.f, sl_ = 0.f, pl = 0.f;
        if (t == Tn - 1 && u == Un - 1) sb = expf(a + lpb[k] - ll);
        if (t < Tn - 1) sb = expf(a + lpb[k] - ll + betas[k + maxU]);
        const bool has_label = u < Un - 1;
        int lab = -1;
        if (has_label) { sl_ = expf(a + lpl[k] - ll + betas[k + maxU + 1]); pl = expf(lpl[k] + occ); lab = labels[(long long)b * (maxU - 1) + u]; }
        float dlb = g * (expf(lpb[k] + occ) - sb), dll = g * (pl - sl_);
        if (has_label && lab == blank) { dlb -= g * sl_; dll = dlb; }    // degenerate: label == blank
        rs = g * exp2f(rowref[row] + (occ - lse[((long long)b * maxT + t) * maxU + u]) * 1.4426950408889634f);
        // cells whose whole gradient row is below 1e-30 contribute nothing: treating them as exactly 0 keeps 1/rs finite
        // (a denormal rs would make it +inf and the patched columns NaN)
        if (!(fabsf(rs) > 1e-30f && fabsf(rs) < CUDART_INF_F)) rs = 0.f;
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

// out[n] += sum_r A[r, n] for a row-major (rows, N) matrix: one block per 32 columns, 8 row lanes, fixed summation order
__global__ void __launch_bounds__(256) colsum_add_kernel(const float* __restrict__ A, long long rows, int N, float* __restrict__ out) {
    __shared__ float part[8][33];
    const int c = threadIdx.x & 31, rl = threadIdx.x >> 5, n = blockIdx.x * 32 + c;
    float acc = 0.f;
    if (n < N)
        for (long long r = rl; r < rows; r += 8) acc += A[r * N + n];
    part[rl][c] = acc;
    __syncthreads();
    if (rl == 0 && n < N) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) s += part[k][c];
        out[n] += s;
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

// out[v] += sum_r x[r,v]   (db of the exact path)
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
