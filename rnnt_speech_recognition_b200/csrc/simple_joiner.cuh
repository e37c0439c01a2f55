// simple_joiner.cuh -- the trivial joiner of pruned RNN-T (Kuang et al., Interspeech 2022), fp32, sm_90a.
//
// Cell (t,u) of utterance b has logits x[v] = am[b,t,v] + lm[b,u,v]: no tanh, no H x V projection.  Its log-softmax
// normaliser factorises: with ma[t] = max_v am[t,v], ml[u] = max_v lm[u,v], Ea = exp(am - ma), El = exp(lm - ml),
//     lse(t,u) = ma[t] + ml[u] + log Nrm[t,u],   Nrm = Ea . El^T      (a (T x V) . (V x U) GEMM per utterance)
// and its logit gradient dx[t,u,v] = G[t,u] Ea[t,v] El[u,v] - (arc terms), G = g exp(alpha + beta - ll - (lse - ma - ml)),
// so that d_am = Ea (.) (G . El) and d_lm = El (.) (G^T . Ea) are two more GEMMs plus sparse arc terms.
//
//   simple_exp_rows_kernel    row maxima and Ea / El (0 on padded rows)
//   bgemm_kernel              batched fp32 FMA GEMM, 128 x 128 x 8 tiles, optional element-wise product in the epilogue
//   simple_lse_kernel         lse and the skewed lp_blank / lp_label planes; a cell whose Nrm < 2^-64 (the factorised sum
//                             has underflowed: am's and lm's large entries lie in different columns) is flagged and gets
//                             its lse by a direct log-sum-exp over V
//   simple_g_kernel           G per cell (0 on padded, flagged and infeasible cells)
//   simple_dam_fix_kernel     per (b,t): the flagged cells' exact softmax terms, then the blank / label arc terms of d_am
//   simple_dlm_fix_kernel     per (b,u): the same for d_lm
//   prune_score_kernel        per (b,t): the band score of every start s and its smallest argmax (fp64 prefix sums)
//   prune_windows_kernel      per b: the monotone / bounded-step scans over t and the per-column frame windows
// No float atomics anywhere: every sum has one writer and a fixed order, so two runs are bit-identical.
#pragma once
#include <climits>

#include "kernels_simt.cuh"

namespace rb {

constexpr float SIMPLE_NRM_MIN = 5.421010862427522e-20f;     // 2^-64: below it the factorised normaliser is not trusted

// One warp per row of x (rows = B * maxR, row stride V): m[row] = max_v x, E[row,:] = exp(x - m).  Rows past the
// utterance's extent (i >= len[b] + extra) get m = 0 and E = 0, so nothing downstream depends on their contents.
__global__ void __launch_bounds__(256) simple_exp_rows_kernel(const float* __restrict__ x, long long rows, int maxR, int V,
                                                              const int* __restrict__ len, int extra,
                                                              float* __restrict__ m, float* __restrict__ E) {
    const long long row = warp_row();
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int b = (int)(row / maxR), i = (int)(row - (long long)b * maxR);
    const float* xr = x + row * (long long)V;
    float* er = E + row * (long long)V;
    if (i >= len[b] + extra) {
        for (int v = lane; v < V; v += 32) er[v] = 0.f;
        if (lane == 0) m[row] = 0.f;
        return;
    }
    float mx = -CUDART_INF_F;
    for (int v = lane; v < V; v += 32) mx = fmaxf(mx, xr[v]);
    mx = warp_max(mx);
    for (int v = lane; v < V; v += 32) er[v] = expf(xr[v] - mx);
    if (lane == 0) m[row] = mx;
}

// C[b] = A[b] . B[b] (EPI == 0) or X[b] (.) (A[b] . B[b]) (EPI == 1, X laid out as C), batch b = blockIdx.z.
// 128 x 128 x 8 tiles, 256 threads, 8 x 8 register micro-tiles from a double-buffered shared-memory stage (the shape of
// sgemm128_kernel), with guarded scalar global accesses so that no dimension or stride has to be a multiple of 4.
// AK: A(m,k) = A[m*sAm + k] (else A[k*sAk + m]); BN: B(k,n) = B[k*sBk + n] (else B[n*sBn + k]).
template <bool AK, bool BN, int EPI>
__global__ void __launch_bounds__(256) bgemm_kernel(const float* __restrict__ A, const float* __restrict__ Bm,
                                                    float* __restrict__ C, const float* __restrict__ X, int M, int N, int K,
                                                    long long sA, long long sB, long long ldc, long long bA, long long bB,
                                                    long long bC) {
    constexpr int BM = 128, BN_ = 128, BK = 8;
    __shared__ __align__(16) float As[2][BK][BM];
    __shared__ __align__(16) float Bs[2][BK][BN_];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN_;
    A += (long long)blockIdx.z * bA;
    Bm += (long long)blockIdx.z * bB;
    C += (long long)blockIdx.z * bC;
    if (EPI) X += (long long)blockIdx.z * bC;
    float ra[4], rb[4];
    auto gload = [&](int k0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (AK) {       // row m = tid/2, k = (tid&1)*4 + j
                const int m = m0 + (tid >> 1), k = k0 + (tid & 1) * 4 + j;
                ra[j] = (m < M && k < K) ? A[(long long)m * sA + k] : 0.f;
            } else {        // k = tid/32, m = (tid&31)*4 + j
                const int k = k0 + (tid >> 5), m = m0 + (tid & 31) * 4 + j;
                ra[j] = (m < M && k < K) ? A[(long long)k * sA + m] : 0.f;
            }
            if (BN) {
                const int k = k0 + (tid >> 5), n = n0 + (tid & 31) * 4 + j;
                rb[j] = (n < N && k < K) ? Bm[(long long)k * sB + n] : 0.f;
            } else {
                const int n = n0 + (tid >> 1), k = k0 + (tid & 1) * 4 + j;
                rb[j] = (n < N && k < K) ? Bm[(long long)n * sB + k] : 0.f;
            }
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (AK) As[buf][(tid & 1) * 4 + j][tid >> 1] = ra[j];
            else As[buf][tid >> 5][(tid & 31) * 4 + j] = ra[j];
            if (BN) Bs[buf][tid >> 5][(tid & 31) * 4 + j] = rb[j];
            else Bs[buf][(tid & 1) * 4 + j][tid >> 1] = rb[j];
        }
    };
    float acc[8][8] = {};
    gload(0);
    sstore(0);
    __syncthreads();
    int buf = 0;
    for (int k0 = 0; k0 < K; k0 += BK) {
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
        for (int j = 0; j < 8; ++j) {
            const int gn = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + j - 4);
            if (gn >= N) continue;
            const long long o = (long long)gm * ldc + gn;
            C[o] = EPI ? X[o] * acc[i][j] : acc[i][j];
        }
    }
}

// Per-cell inputs of the simple lattice's planes: the cell, its logits' row pointers and its maxima.
struct SimpleCell {
    const float *a, *l;      // am[b,t,:], lm[b,u,:]
    float ma, ml;
};
__device__ __forceinline__ SimpleCell simple_cell(const RowCell& c, const float* am, const float* lm, const float* ma,
                                                  const float* ml, int maxT, int maxU, int V) {
    const long long ra = (long long)c.b * maxT + c.t, rl = (long long)c.b * maxU + c.u;
    return {am + ra * V, lm + rl * V, ma[ra], ml[rl]};
}

// log sum_v exp(am[t,v] + lm[u,v]) over V, by one warp (the underflow fallback; every lane returns the value)
__device__ __forceinline__ float direct_lse(const SimpleCell& s, int V, int lane) {
    float mx = -CUDART_INF_F;
    for (int v = lane; v < V; v += 32) mx = fmaxf(mx, s.a[v] + s.l[v]);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int v = lane; v < V; v += 32) sum += expf(s.a[v] + s.l[v] - mx);
    return mx + logf(warp_sum(sum));
}

// One warp per lattice cell: lse = ma + ml + log Nrm (or the direct sum when Nrm < 2^-64, flag = 1), and the skewed
// lp_blank / lp_label planes the alpha/beta wavefront reads.  Padded cells: flag = 0, nothing else written.
__global__ void __launch_bounds__(256) simple_lse_kernel(const float* __restrict__ am, const float* __restrict__ lm,
                                                         const float* __restrict__ ma, const float* __restrict__ ml,
                                                         const float* __restrict__ nrm, const int* __restrict__ xlen,
                                                         const int* __restrict__ ylen, const int* __restrict__ labels,
                                                         int maxT, int maxU, long long SK, long long ncells, int V,
                                                         int blank, float* __restrict__ lse, float* __restrict__ lpb,
                                                         float* __restrict__ lpl, unsigned char* __restrict__ flag) {
    const long long cell = warp_row();
    const int lane = threadIdx.x & 31;
    if (cell >= ncells) return;
    const RowCell c = row_cell(cell, maxT, maxU, xlen, ylen);
    if (c.padded()) {
        if (lane == 0) flag[cell] = 0;
        return;
    }
    const SimpleCell s = simple_cell(c, am, lm, ma, ml, maxT, maxU, V);
    const float n = nrm[cell];
    const bool under = !(n >= SIMPLE_NRM_MIN);
    const float l = under ? direct_lse(s, V, lane) : s.ma + s.ml + logf(n);
    if (lane == 0) {
        flag[cell] = under ? 1 : 0;
        lse[cell] = l;
        const long long k = c.sk(maxU, SK);
        lpb[k] = s.a[blank] + s.l[blank] - l;
        if (c.u < c.Un - 1) {
            const int y = c.label(labels, maxU);
            lpl[k] = s.a[y] + s.l[y] - l;
        }
    }
}

// G[cell] = g * exp(alpha + beta - ll - (lse - ma - ml)) on the cells whose softmax the GEMMs carry, 0 elsewhere.
__global__ void __launch_bounds__(256) simple_g_kernel(const float* __restrict__ ma, const float* __restrict__ ml,
                                                       const float* __restrict__ lse, const float* __restrict__ alphas,
                                                       const float* __restrict__ betas, const float* __restrict__ llf,
                                                       const unsigned char* __restrict__ flag, const float* __restrict__ gc,
                                                       const int* __restrict__ xlen, const int* __restrict__ ylen,
                                                       int maxT, int maxU, long long SK, long long ncells,
                                                       float* __restrict__ G) {
    const long long cell = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (cell >= ncells) return;
    const RowCell c = row_cell(cell, maxT, maxU, xlen, ylen);
    float v = 0.f;
    const float ll = c.padded() ? 0.f : llf[c.b];
    if (!c.padded() && !flag[cell] && ll > -CUDART_INF_F) {
        const long long k = c.sk(maxU, SK);
        const float g = gc ? gc[c.b] : 1.f;
        const float rel = lse[cell] - ma[(long long)c.b * maxT + c.t] - ml[(long long)c.b * maxU + c.u];
        v = g * expf(alphas[k] + betas[k] - ll - rel);
    }
    G[cell] = v;
}

// The arc occupancies of a valid cell without grad_costs (arc_terms of the loss op, lambda = 0): blank (incl. the
// terminating blank of the last cell) and label.
struct Occ { float b, l; };
__device__ __forceinline__ Occ simple_occ(int b, int t, int u, int Tn, int Un, int maxU, long long SK, const float* lpb,
                                          const float* lpl, const float* alphas, const float* betas, float ll) {
    const long long k = sk_index(b, t, u, maxU, SK);
    const bool has_label = u < Un - 1;
    const ArcTerms<float> arc = arc_terms<float>(alphas[k], ll, lpb[k], has_label ? lpl[k] : 0.f, betas + k, maxU,
                                                 t == Tn - 1 && u == Un - 1, t < Tn - 1, has_label, 0.f);
    return {arc.sb, arc.sl};
}

// Block-wide sum of one float per thread, in a fixed order (warp trees, then warp 0 over the warp sums).
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    float r = 0.f;
    if (w == 0) {
        r = lane < nw ? red[lane] : 0.f;
        r = warp_sum(r);
    }
    return r;      // thread 0 holds the sum
}

constexpr int SIMPLE_FIX_THREADS = 256;

// One block per d_am row (b,t), t < T_b.  1) each flagged cell (t,u), in u order, adds its exact softmax term
// g occ(t,u) softmax(am[t] + lm[u])[v]; 2) d_am[t,blank] -= g sum_u gamma_B(t,u); 3) d_am[t,y_u] -= g gamma_L(t,u): the
// first u of each distinct label sums that label's terms in u order, so each column has one writer.
__global__ void __launch_bounds__(SIMPLE_FIX_THREADS) simple_dam_fix_kernel(
    const float* __restrict__ am, const float* __restrict__ lm, const float* __restrict__ lse, const float* __restrict__ lpb,
    const float* __restrict__ lpl, const float* __restrict__ alphas, const float* __restrict__ betas,
    const float* __restrict__ llf, const unsigned char* __restrict__ flag, const float* __restrict__ gc,
    const int* __restrict__ xlen, const int* __restrict__ ylen, const int* __restrict__ labels, int maxT, int maxU,
    long long SK, int V, int blank, float* __restrict__ d_am) {
    __shared__ float gl[1024];
    __shared__ int lab[1024];
    __shared__ float red[32];
    const int b = blockIdx.x / maxT, t = blockIdx.x - b * maxT, tid = threadIdx.x;
    const int Tn = xlen[b], Un = ylen[b] + 1;
    const float ll = llf[b];
    if (t >= Tn || !(ll > -CUDART_INF_F)) return;
    const float g = gc ? gc[b] : 1.f;
    float* row = d_am + ((long long)b * maxT + t) * V;
    const float* a = am + ((long long)b * maxT + t) * V;
    const long long c0 = ((long long)b * maxT + t) * maxU;
    int any = 0;                                   // most rows have no flagged cell: skip the ordered walk over u
    for (int u = tid; u < Un; u += SIMPLE_FIX_THREADS) any |= flag[c0 + u];
    if (__syncthreads_or(any)) {
        for (int u = 0; u < Un; ++u) {
            if (!flag[c0 + u]) continue;
            const long long k = sk_index(b, t, u, maxU, SK);
            const float occ = g * expf(alphas[k] + betas[k] - ll), l = lse[c0 + u];
            const float* lr = lm + ((long long)b * maxU + u) * V;
            for (int v = tid; v < V; v += SIMPLE_FIX_THREADS) row[v] += occ * expf(a[v] + lr[v] - l);
        }
    }
    float sb = 0.f;
    for (int u = tid; u < Un; u += SIMPLE_FIX_THREADS) {
        const Occ o = simple_occ(b, t, u, Tn, Un, maxU, SK, lpb, lpl, alphas, betas, ll);
        sb += o.b;
        gl[u] = o.l;
        lab[u] = u < Un - 1 ? labels[(long long)b * (maxU - 1) + u] : -1;
    }
    sb = block_sum(sb, red);          // (its barriers also order the flagged cells' writes before the arc terms)
    if (tid == 0) row[blank] -= g * sb;
    __syncthreads();
    for (int u = tid; u < Un - 1; u += SIMPLE_FIX_THREADS) {
        const int y = lab[u];
        bool first = true;
        for (int j = 0; j < u && first; ++j) first = lab[j] != y;
        if (!first) continue;
        float s = 0.f;
        for (int j = u; j < Un - 1; ++j)
            if (lab[j] == y) s += gl[j];
        row[y] -= g * s;
    }
}

// One block per d_lm row (b,u), u < U_b: the flagged cells (t,u) in t order, then d_lm[u,blank] -= g sum_t gamma_B and
// d_lm[u,y_u] -= g sum_t gamma_L (in this order, so a label equal to blank is applied after the blank term).
__global__ void __launch_bounds__(SIMPLE_FIX_THREADS) simple_dlm_fix_kernel(
    const float* __restrict__ am, const float* __restrict__ lm, const float* __restrict__ lse, const float* __restrict__ lpb,
    const float* __restrict__ lpl, const float* __restrict__ alphas, const float* __restrict__ betas,
    const float* __restrict__ llf, const unsigned char* __restrict__ flag, const float* __restrict__ gc,
    const int* __restrict__ xlen, const int* __restrict__ ylen, const int* __restrict__ labels, int maxT, int maxU,
    long long SK, int V, int blank, float* __restrict__ d_lm) {
    __shared__ float red[32];
    const int b = blockIdx.x / maxU, u = blockIdx.x - b * maxU, tid = threadIdx.x;
    const int Tn = xlen[b], Un = ylen[b] + 1;
    const float ll = llf[b];
    if (u >= Un || !(ll > -CUDART_INF_F)) return;
    const float g = gc ? gc[b] : 1.f;
    float* row = d_lm + ((long long)b * maxU + u) * V;
    const float* lr = lm + ((long long)b * maxU + u) * V;
    int any = 0;                                   // most rows have no flagged cell: skip the ordered walk over t
    for (int t = tid; t < Tn; t += SIMPLE_FIX_THREADS) any |= flag[((long long)b * maxT + t) * maxU + u];
    if (__syncthreads_or(any)) {
        for (int t = 0; t < Tn; ++t) {
            const long long c = ((long long)b * maxT + t) * maxU + u;
            if (!flag[c]) continue;
            const long long k = sk_index(b, t, u, maxU, SK);
            const float occ = g * expf(alphas[k] + betas[k] - ll), l = lse[c];
            const float* a = am + ((long long)b * maxT + t) * V;
            for (int v = tid; v < V; v += SIMPLE_FIX_THREADS) row[v] += occ * expf(a[v] + lr[v] - l);
        }
    }
    float sb = 0.f, sl = 0.f;
    for (int t = tid; t < Tn; t += SIMPLE_FIX_THREADS) {
        const Occ o = simple_occ(b, t, u, Tn, Un, maxU, SK, lpb, lpl, alphas, betas, ll);
        sb += o.b;
        sl += o.l;
    }
    sb = block_sum(sb, red);
    sl = block_sum(sl, red);
    if (tid == 0) {
        row[blank] -= g * sb;
        if (u < Un - 1) row[labels[(long long)b * (maxU - 1) + u]] -= g * sl;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Band policy (DESIGN §1), per utterance with S = s_range:
//   score(t,s) = sum_{u=s}^{min(s+S,U_b)-1} gamma_B(t,u) - gamma_L(t,s-1),  s in [0, max(0, U_b - S)],  gamma_L(t,-1) = 0
//   raw s_t = smallest argmax (t < T_b - 1), s_{T_b-1} = max(0, U_b - S); then the two scans over t of prune_windows.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int PRUNE_WARPS = 4;

// One warp per frame t < T_b: gamma_B(t,.) summed into an fp64 prefix (a difference of fp32 prefix sums would cancel),
// then every start s scored from it and the smallest argmax written to s_raw[b,t].
__global__ void __launch_bounds__(PRUNE_WARPS * 32) prune_score_kernel(
    const float* __restrict__ lpb, const float* __restrict__ lpl, const float* __restrict__ alphas,
    const float* __restrict__ betas, const float* __restrict__ llf, const int* __restrict__ xlen,
    const int* __restrict__ ylen, int maxT, int maxU, long long SK, int S, int* __restrict__ s_raw) {
    __shared__ double P[PRUNE_WARPS][1025];
    const int b = blockIdx.x, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.y * PRUNE_WARPS + w;
    const int Tn = xlen[b], Un = ylen[b] + 1;
    if (t >= Tn) return;
    const int smax = max(0, Un - S);
    int* out = s_raw + (long long)b * maxT + t;
    if (t == Tn - 1) {
        if (lane == 0) *out = smax;
        return;
    }
    const float ll = llf[b];
    const bool ok = ll > -CUDART_INF_F;
    double* p = P[w];
    double carry = 0.0;
    if (lane == 0) p[0] = 0.0;
    for (int u0 = 0; u0 < Un; u0 += 32) {
        const int u = u0 + lane;
        double x = (ok && u < Un) ? (double)simple_occ(b, t, u, Tn, Un, maxU, SK, lpb, lpl, alphas, betas, ll).b : 0.0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (u < Un) p[u + 1] = carry + x;
        carry += __shfl_sync(0xffffffffu, x, 31);
    }
    __syncwarp();
    double best = -1e300;
    int bs = 0;
    for (int s = lane; s <= smax; s += 32) {
        double sc = p[min(s + S, Un)] - p[s];
        if (s > 0 && ok) sc -= (double)simple_occ(b, t, s - 1, Tn, Un, maxU, SK, lpb, lpl, alphas, betas, ll).l;
        if (sc > best) { best = sc; bs = s; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int os = __shfl_xor_sync(0xffffffffu, bs, o);
        if (ob > best || (ob == best && os < bs)) { best = ob; bs = os; }
    }
    if (lane == 0) *out = bs;
}

constexpr int PRUNE_CHUNK = 4096, PRUNE_THREADS = 256;

// One block per utterance.  From t = T_b - 1 down, in one pass:
//   m_t = min_{t' >= t} s_raw[t']                                   (monotone)
//   q_t = max_{t' >= t} (m_{t'} - (S-1) t'),  s_t = min((S-1) t, (S-1) t + q_t)   (bounded step, start at 0)
// then for each column u < U_b the frames t with s_t <= u < s_t + S, an interval [c_u, a_u) because s is non-decreasing:
// a_u = #{t : s_t <= u}, c_u = #{t : s_t <= u - S}.  Empty intervals and columns u >= U_b get (0, -1).
__global__ void __launch_bounds__(PRUNE_THREADS) prune_windows_kernel(const int* __restrict__ s_raw, int* __restrict__ s_band,
                                                                     const int* __restrict__ xlen, const int* __restrict__ ylen,
                                                                     int maxT, int maxU, int S, int* __restrict__ t_lo,
                                                                     int* __restrict__ t_hi) {
    __shared__ int sm[PRUNE_CHUNK];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int Tn = xlen[b], Un = ylen[b] + 1;
    const int* sr = s_raw + (long long)b * maxT;
    int* sb = s_band + (long long)b * maxT;
    const long long step = S - 1;
    int m = INT_MAX;
    long long q = LLONG_MIN;
    for (int hi = Tn; hi > 0; hi -= PRUNE_CHUNK) {           // chunks [lo, hi) from the end
        const int lo = max(0, hi - PRUNE_CHUNK);
        for (int t = lo + tid; t < hi; t += PRUNE_THREADS) sm[t - lo] = sr[t];
        __syncthreads();
        if (tid == 0) {
            for (int t = hi - 1; t >= lo; --t) {
                m = min(m, sm[t - lo]);
                q = max(q, (long long)m - step * t);
                const long long a = step * t;
                sm[t - lo] = (int)min(a, a + q);
            }
        }
        __syncthreads();
        for (int t = lo + tid; t < hi; t += PRUNE_THREADS) sb[t] = sm[t - lo];
        __syncthreads();
    }
    for (int u = tid; u < maxU; u += PRUNE_THREADS) {
        int lo = 0, hi = -1;
        if (u < Un && Tn > 0) {
            auto count_le = [&](long long x) {          // #{t < T_b : s_t <= x}
                int l = 0, h = Tn;
                while (l < h) {
                    const int mid = (l + h) >> 1;
                    if (sb[mid] <= x) l = mid + 1; else h = mid;
                }
                return l;
            };
            const int a = count_le(u), c = count_le((long long)u - S);
            if (c <= a - 1) { lo = c; hi = a - 1; }
        }
        t_lo[(long long)b * maxU + u] = lo;
        t_hi[(long long)b * maxU + u] = hi;
    }
}

}  // namespace rb
