// joint_step.cuh -- the greedy-decode joint (SURVEY 8 f2; reference utils/decoding.py:6-18, called per decode step at
// utils/decoding.py:69-78): ONE lattice cell per batch row,
//     logits[b,:] = tanh((f[b,:] + g[b,:]) . K1 + b1) . K2 + b2,   best[b] = argmax_v,   best_logp[b] = log_softmax[best]
// as ONE launch with the argmax / log-softmax in its epilogue (the reference materialises (B,1,1,P), (B,1,1,H) and
// (B,1,1,V) tensors through two Keras Dense layers, then log_softmax, then argmax).  fp32 FMA arithmetic: this is
// inference, the prediction must be the reference's.
//
// A decode step is latency bound (B is 1 in the reference's greedy decoder): the work of one batch row is spread over a
// thread-block CLUSTER of 8 CTAs -- each computes an eighth of the hidden units, the slices are exchanged through
// distributed shared memory, each CTA then owns an eighth of the vocabulary and the (max, argmax, sum-exp) partials
// are combined in the leader's shared memory.  No global scratch, no second launch.
#pragma once
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <math_constants.h>

namespace rb {

constexpr int STEP_CLUSTER = 8;
constexpr int STEP_THREADS = 256;
constexpr int STEP_MAX_DIM = 4096;     // P, H <= 4096 (shared-memory staging of the input row and the hidden row)
// Shared memory per CTA: the static part_m / part_s / part_i below plus the dynamic joint_step_smem().  Together they may
// reach 48 KB by default and the sm_90 opt-in ceiling of 227 KB with cudaFuncAttributeMaxDynamicSharedMemorySize.
constexpr size_t STEP_STATIC_SMEM = STEP_CLUSTER * (2 * sizeof(float) + sizeof(int));
constexpr size_t STEP_SMEM_DEFAULT = 48 * 1024 - STEP_STATIC_SMEM;    // largest dynamic size without the opt-in
constexpr size_t STEP_SMEM_MAX = 232448 - STEP_STATIC_SMEM;           // largest dynamic size with it

// Argmax order of the decode step: a NaN outranks every number (the first NaN wins, as np.argmax / torch.argmax), and
// among equal values the smaller index wins (as tf.argmax).  Is (c, ic) ahead of (a, ia)?
__device__ __forceinline__ bool step_argmax_before(float c, int ic, float a, int ia) {
    if (c != c) return a == a || ic < ia;
    return c > a || (c == a && ic < ia);
}

struct StepParams {
    const float* f; const float* g;     // (B, P) rows with strides ldf / ldg
    long long ldf, ldg;
    const float* K1; const float* b1;   // (P, H), (H)   -- K1 == NULL: f, g are the already-projected activations (P == H)
    const float* K2; const float* b2;   // (H, V), (V)
    int B, P, H, V;
    float* logits;                      // (B, V) or NULL
    int* best;                          // (B) or NULL
    float* best_logp;                   // (B) or NULL
};

__global__ void __cluster_dims__(STEP_CLUSTER, 1, 1) __launch_bounds__(STEP_THREADS) joint_step_kernel(const StepParams p) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned rank = cluster.block_rank();
    const int b = blockIdx.x / STEP_CLUSTER, tid = threadIdx.x;
    extern __shared__ float sm[];
    float* x = sm;                       // [max(P, STEP_THREADS)]  f + g (later: int scratch of the argmax)
    float* z = sm + (p.P > STEP_THREADS ? p.P : STEP_THREADS);   // [H]  tanh(...)  (own slice first, then the whole row)
    float* red = z + p.H;                // [STEP_THREADS] scratch
    __shared__ float part_m[STEP_CLUSTER], part_s[STEP_CLUSTER];
    __shared__ int part_i[STEP_CLUSTER];

    for (int i = tid; i < p.P; i += STEP_THREADS) x[i] = p.f[(long long)b * p.ldf + i] + p.g[(long long)b * p.ldg + i];
    __syncthreads();

    // ---- stage 1: this CTA's slice of the hidden units
    const int hs = (p.H + STEP_CLUSTER - 1) / STEP_CLUSTER, h0 = rank * hs, hn = min(hs, p.H - h0);
    if (p.K1) {
        // threads = (column of the slice) x (partition of the P reduction); partial sums combined through shared memory
        const int cols = hn > 0 ? hn : 1, parts = max(1, STEP_THREADS / cols);
        const int c = tid % cols, pg = tid / cols;
        float acc = 0.f;
        if (hn > 0 && pg < parts) {
            const int per = (p.P + parts - 1) / parts, pb = pg * per, pe = min(p.P, pb + per);
            const float* k = p.K1 + h0 + c;
            for (int i = pb; i < pe; ++i) acc = fmaf(x[i], __ldg(k + (long long)i * p.H), acc);
        }
        red[tid] = (hn > 0 && pg < parts) ? acc : 0.f;
        __syncthreads();
        if (tid < hn) {
            float s = p.b1 ? __ldg(p.b1 + h0 + tid) : 0.f;
            for (int q = 0; q < parts; ++q) s += red[q * cols + tid];
            z[h0 + tid] = tanhf(s);
        }
    } else {
        for (int i = tid; i < hn; i += STEP_THREADS) z[h0 + i] = tanhf(x[h0 + i]);
    }
    cluster.sync();
    // gather the other CTAs' slices through distributed shared memory
    for (unsigned r = 0; r < STEP_CLUSTER; ++r) {
        if (r == rank) continue;
        const float* rz = cluster.map_shared_rank(z, r);
        const int r0 = r * hs, rn = min(hs, p.H - r0);
        for (int i = tid; i < rn; i += STEP_THREADS) z[r0 + i] = rz[r0 + i];
    }
    cluster.sync();

    // ---- stage 2: this CTA's slice of the vocabulary (its logits stay in shared memory for the two reductions)
    const int vs = (p.V + STEP_CLUSTER - 1) / STEP_CLUSTER, v0 = rank * vs, vn = max(0, min(vs, p.V - v0));
    float* lg = red + STEP_THREADS;       // [vs]
    {
        const int cols = vn > 0 ? min(vn, STEP_THREADS) : 1, parts = max(1, STEP_THREADS / cols);
        for (int vb = 0; vb < vn; vb += cols) {            // (slices wider than the block: several passes)
            const int c = tid % cols, pg = tid / cols, v = v0 + vb + c;
            float acc = 0.f;
            const bool on = (vb + c) < vn && pg < parts;
            if (on) {
                const int per = (p.H + parts - 1) / parts, hb = pg * per, he = min(p.H, hb + per);
                const float* k = p.K2 + v;
                for (int i = hb; i < he; ++i) acc = fmaf(z[i], __ldg(k + (long long)i * p.V), acc);
            }
            __syncthreads();
            red[tid] = on ? acc : 0.f;
            __syncthreads();
            if (tid < cols && (vb + tid) < vn) {
                float s = p.b2 ? __ldg(p.b2 + v0 + vb + tid) : 0.f;
                for (int q = 0; q < parts; ++q) s += red[q * cols + tid];
                lg[vb + tid] = s;
                if (p.logits) p.logits[(long long)b * p.V + v0 + vb + tid] = s;
            }
        }
    }
    __syncthreads();
    // slice max / argmax in the order of step_argmax_before, then sum of exp against the slice max.  Each thread starts
    // from its first element, so a slice of -inf still yields one of its indices; (-inf, INT_MAX) stands for a thread
    // (or CTA) that owns no element and loses to every element.
    float my = -CUDART_INF_F; int myi = 0x7fffffff;
    if (tid < vn) { my = lg[tid]; myi = v0 + tid; }
    for (int i = tid + STEP_THREADS; i < vn; i += STEP_THREADS)
        if (step_argmax_before(lg[i], v0 + i, my, myi)) { my = lg[i]; myi = v0 + i; }
    int* redi = reinterpret_cast<int*>(x);                  // (the input row is dead: reuse it; P >= 1 ... see launcher: smem has room)
    red[tid] = my; redi[tid] = myi;
    __syncthreads();
    for (int o = STEP_THREADS / 2; o > 0; o >>= 1) {
        if (tid < o) {
            const float a2 = red[tid], c2 = red[tid + o];
            const int ia = redi[tid], ic = redi[tid + o];
            if (step_argmax_before(c2, ic, a2, ia)) { red[tid] = c2; redi[tid] = ic; }
        }
        __syncthreads();
    }
    const float bm = red[0];
    const int bi = redi[0];
    __syncthreads();
    float ssum = 0.f;                                       // (a slice of -inf adds nothing: not exp(-inf - -inf) = NaN)
    if (bm != -CUDART_INF_F)
        for (int i = tid; i < vn; i += STEP_THREADS) ssum += expf(lg[i] - bm);
    red[tid] = ssum;
    __syncthreads();
    for (int o = STEP_THREADS / 2; o > 0; o >>= 1) {
        if (tid < o) red[tid] += red[tid + o];
        __syncthreads();
    }
    // ---- combine the eight slices in the leader's shared memory
    if (tid == 0) {
        float* lm = cluster.map_shared_rank(part_m, 0);
        float* ls = cluster.map_shared_rank(part_s, 0);
        int* li = cluster.map_shared_rank(part_i, 0);
        lm[rank] = vn > 0 ? bm : -CUDART_INF_F; ls[rank] = vn > 0 ? red[0] : 0.f; li[rank] = bi;
    }
    cluster.sync();
    if (rank == 0 && tid == 0) {
        float M = -CUDART_INF_F; int I = 0x7fffffff;
        for (int r = 0; r < STEP_CLUSTER; ++r)
            if (step_argmax_before(part_m[r], part_i[r], M, I)) { M = part_m[r]; I = part_i[r]; }
        float S = 0.f;
        for (int r = 0; r < STEP_CLUSTER; ++r) S += part_s[r] * expf(part_m[r] - M);
        if (p.best) p.best[b] = I;
        if (p.best_logp) p.best_logp[b] = -logf(S);          // log_softmax at the maximum: M - (M + log S)
    }
    // (the leader's shared memory must outlive the remote writes: every CTA passed the cluster barrier above)
}

inline size_t joint_step_smem(int P, int H, int V) {
    const int vs = (V + STEP_CLUSTER - 1) / STEP_CLUSTER;
    const int xs = P > STEP_THREADS ? P : STEP_THREADS;      // the input row is reused as the int scratch of the argmax
    return sizeof(float) * ((size_t)xs + H + STEP_THREADS + vs);
}

// Largest V whose joint_step_smem() fits STEP_SMEM_MAX (P, H within their limits): 8 (58088 - max(P,256) - H - 256).
inline int joint_step_max_v(int P, int H) {
    const int xs = P > STEP_THREADS ? P : STEP_THREADS;
    return STEP_CLUSTER * ((int)(STEP_SMEM_MAX / sizeof(float)) - xs - H - STEP_THREADS);
}

}  // namespace rb
