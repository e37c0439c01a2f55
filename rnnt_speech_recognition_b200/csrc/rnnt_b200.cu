// rnnt_b200.cu -- C ABI (include/rnnt_b200.h) and host-side orchestration of the RNN-T loss hot
// path on H100 (sm_90a).  No allocation, no host synchronisation (except the reference-mandated one in
// compute_rnnt_loss), everything stream-ordered on the caller's stream.
#include "../../include/rnnt_b200.h"

#include <atomic>
#include <climits>
#include <cstdio>
#include <cstdint>
#include <cfloat>
#include <cmath>
#include <vector>

#include <cuda_runtime.h>

#include "kernels_simt.cuh"
#include "simple_joiner.cuh"
#include "timing.cuh"
#include "joint_step.cuh"
#ifndef RNNTB200_NO_TC
#include "joint_tc.cuh"
#endif

namespace {

std::atomic<unsigned long long> g_launches{0};
#define RB_LAUNCHED(n) g_launches.fetch_add((n), std::memory_order_relaxed)

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
inline long long skew_plane(int maxT, int maxU) { return (long long)(maxT + maxU - 1) * maxU; }

// Workspace of the loss op proper (shared by compute_rnnt_loss and the joint path).
template <typename T>
struct LossWs {
    T *lpb, *lpl, *alphas, *betas, *lse, *llf, *llb;
    size_t bytes;
    LossWs(void* base, int B, int maxT, int maxU) {
        const size_t SK = (size_t)skew_plane(maxT, maxU), N = (size_t)maxT * maxU;
        T* p = reinterpret_cast<T*>(base);
        lpb = p; p += B * SK;
        lpl = p; p += B * SK;
        alphas = p; p += B * SK;
        betas = p; p += B * SK;
        lse = p; p += B * N;
        llf = p; p += B;
        llb = p; p += B;
        bytes = (size_t)B * (4 * SK + N + 2) * sizeof(T);
    }
};

// costs[b] = -llForward[b] (cpu_rnnt.h:172), with the reference's consistency guard of the two lattice passes
// (cpu_rnnt.h:166-170: "WARNING: Forward backward likelihood mismatch" when |llForward - llBackward| > 0.1) as a
// device-side printf: stream-ordered, costs nothing unless it fires, and needs no read-back.
__global__ void finish_costs_kernel(const float* __restrict__ llf, const float* __restrict__ llb, float* __restrict__ out, int n,
                                    const int* __restrict__ overflow) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (overflow && *overflow) { out[i] = __int_as_float(0x7fc00000); return; }   // broken valid_tile_bound promise (tile_compact_kernel reported it)
    out[i] = -llf[i];
    const float diff = fabsf(llf[i] - llb[i]);
    if (diff > 0.1f) printf("WARNING: Forward backward likelihood mismatch %f (utterance %d)\n", diff, i);
}

// The windows of the alignment-restricted entries (rb::Windows); the entries without them pass none.  Both pointers or
// neither: exactly one NULL is an argument error.
constexpr rb::Windows no_windows{nullptr, nullptr};
inline bool windows_ok(const int* t_lo, const int* t_hi) { return (t_lo == nullptr) == (t_hi == nullptr); }

inline rnntStatus_t check_launch() { return cudaGetLastError() == cudaSuccess ? RNNT_STATUS_SUCCESS : RNNT_STATUS_EXECUTION_FAILED; }

// overflow (nullable): the tensor-core forward's broken valid_tile_bound word, which turns the costs into NaN
rnntStatus_t launch_finish_costs(const float* llf, const float* llb, float* costs, int B, const int* overflow, cudaStream_t s) {
    finish_costs_kernel<<<(B + 127) / 128, 128, 0, s>>>(llf, llb, costs, B, overflow);
    RB_LAUNCHED(1);
    return check_launch();
}

template <typename T>
rnntStatus_t launch_alpha_beta(const LossWs<T>& w, const int* xlen, const int* ylen, int B, int maxT, int maxU,
                               cudaStream_t s, const rb::Windows& win = no_windows) {
    const int threads = (maxU + 31) / 32 * 32;
    constexpr int PF = sizeof(T) == 4 ? 8 : 4;
    rb::ScopedTimer tm("alpha_beta_kernel", s);
    if constexpr (sizeof(T) == 4) {
        if (win.lo)
            rb::alpha_beta_windowed_kernel<PF><<<dim3(B, 2), threads, 0, s>>>(w.lpb, w.lpl, w.alphas, w.betas, w.llf, w.llb,
                                                                              xlen, ylen, maxU, skew_plane(maxT, maxU), win);
    }
    if (sizeof(T) != 4 || !win.lo)
        rb::alpha_beta_kernel<T, PF><<<dim3(B, 2), threads, 0, s>>>(w.lpb, w.lpl, w.alphas, w.betas, w.llf, w.llb, xlen,
                                                                    ylen, maxU, skew_plane(maxT, maxU));
    RB_LAUNCHED(1);
    return check_launch();
}

// Forced alignment over the lp_blank / lp_label planes of a finished forward: the Viterbi wavefront, then the backtrace.
// The costs are final by now (finish_costs_kernel ran), so the decision bit-plane, (maxT+maxU-1) * ceil(maxU/32) words
// per utterance, goes into the beta plane ((maxT+maxU-1) * maxU floats) and delta's end value into llb: the workspace
// keeps its size, and cannot feed a backward call afterwards.
rnntStatus_t launch_align(const LossWs<float>& w, const int* xlen, const int* ylen, int B, int maxT, int maxU,
                          const int* overflow, float* best_logp, int* frames, cudaStream_t s) {
    unsigned* dec = reinterpret_cast<unsigned*>(w.betas);
    {
        rb::ScopedTimer tm("viterbi_kernel", s);
        rb::viterbi_kernel<8><<<B, (maxU + 31) / 32 * 32, 0, s>>>(w.lpb, w.lpl, dec, w.llb, xlen, ylen, maxU,
                                                                  skew_plane(maxT, maxU));
    }
    RB_LAUNCHED(1);
    if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    {
        rb::ScopedTimer tm("backtrace_kernel", s);
        rb::backtrace_kernel<<<B, rb::BT_THREADS, 0, s>>>(dec, w.llb, overflow, xlen, ylen, maxT, maxU, best_logp, frames);
    }
    RB_LAUNCHED(1);
    return check_launch();
}

// argument checks the three align entries add to those of their forward entries
inline bool align_args_ok(const float* best_logp, const int* frames, int maxU) { return best_logp && (frames || maxU == 1); }

// The 16-byte fast paths need float workspace arithmetic, V a multiple of the elements per 16 bytes and 16-byte
// aligned tensors (rows then stay aligned).
template <typename T, typename X>
bool vec_ok(const X* acts, const X* grads, int V) {
    return sizeof(T) == 4 && (V % (16 / (int)sizeof(X))) == 0 && ((uintptr_t)acts % 16) == 0 &&
           (!grads || ((uintptr_t)grads % 16) == 0);
}

// loss op on materialised logits, forward half: lse+gather -> alpha/beta.  costs stay on device in w.llf.
// X is the logits' element type: T itself, or fp16 / bf16 over a float workspace.
template <typename T, typename X>
rnntStatus_t loss_planes(const X* acts, bool vec, const int* labels, const int* ylen, const int* xlen, int V, int B,
                         int maxT, int maxU, int blank, void* workspace, cudaStream_t s,
                         const rb::Windows& win = no_windows) {
    if (maxU > 1024) {
        fprintf(stderr, "rnnt_b200: maxU=%d exceeds the 1024 label positions per utterance limit\n", maxU);
        return RNNT_STATUS_INVALID_VALUE;
    }
    LossWs<T> w(workspace, B, maxT, maxU);
    const long long N = (long long)B * maxT * maxU, SK = skew_plane(maxT, maxU);
    const unsigned blocks = (unsigned)((N * 32 + 255) / 256);
    {
        rb::ScopedTimer tm("lse_gather_kernel", s);
        if constexpr (sizeof(T) == 4) {
            if (vec) {
                if (V <= 8 * 32 * (16 / (int)sizeof(X)))      // 8 pieces of 16 bytes per lane held in registers
                    rb::lse_gather_vec_kernel<X, 8><<<blocks, 256, 0, s>>>(acts, 0, N, V, xlen, ylen, labels, maxT, maxU, SK,
                                                                           blank, w.lse, w.lpb, w.lpl, win);
                else
                    rb::lse_gather_vec_kernel<X, 0><<<blocks, 256, 0, s>>>(acts, 0, N, V, xlen, ylen, labels, maxT, maxU, SK,
                                                                           blank, w.lse, w.lpb, w.lpl, win);
            }
        }
        if (!vec)
            rb::lse_gather_kernel<T, X><<<blocks, 256, 0, s>>>(acts, 0, N, V, xlen, ylen, labels, maxT, maxU, SK, blank,
                                                               w.lse, w.lpb, w.lpl, win);
    }
    RB_LAUNCHED(1);
    if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    if (launch_alpha_beta(w, xlen, ylen, B, maxT, maxU, s, win)) return RNNT_STATUS_EXECUTION_FAILED;
    return RNNT_STATUS_SUCCESS;
}

// backward half: gradients w.r.t. the logits from the planes loss_planes left in the workspace
template <typename T, typename X>
rnntStatus_t loss_grads(const X* acts, X* grads, bool vec, const int* labels, const int* ylen, const int* xlen,
                        const T* gscale, int V, int B, int maxT, int maxU, int blank, void* workspace, cudaStream_t s,
                        float fastemit_lambda, const rb::Windows& win = no_windows) {
    LossWs<T> w(workspace, B, maxT, maxU);
    const long long N = (long long)B * maxT * maxU, SK = skew_plane(maxT, maxU);
    const unsigned blocks = (unsigned)((N * 32 + 255) / 256);
    rb::ScopedTimer tm("rnnt_grad_kernel", s);
    if constexpr (sizeof(T) == 4) {
        if (vec)
            rb::rnnt_grad_vec_kernel<X><<<blocks, 256, 0, s>>>(acts, grads, 0, N, V, xlen, ylen, labels, maxT, maxU, SK, blank,
                                                               w.lse, w.alphas, w.betas, w.llf, gscale, fastemit_lambda, win);
    }
    if (!vec)
        rb::rnnt_grad_kernel<T, X><<<blocks, 256, 0, s>>>(acts, grads, 0, N, V, xlen, ylen, labels, maxT, maxU, SK,
                                                          blank, w.lse, w.alphas, w.betas, w.llf, gscale, fastemit_lambda, win);
    RB_LAUNCHED(1);
    return check_launch();
}

// forward of the device-costs entries (fp32 or 16-bit logits over a float workspace): planes, then the costs
template <typename X>
rnntStatus_t loss_forward(const X* acts, bool vec, const int* labels, const int* ylen, const int* xlen, int V, int B,
                          int maxT, int maxU, int blank, float* costs, void* workspace, cudaStream_t s,
                          const rb::Windows& win = no_windows) {
    rnntStatus_t st = loss_planes<float, X>(acts, vec, labels, ylen, xlen, V, B, maxT, maxU, blank, workspace, s, win);
    if (st) return st;
    const LossWs<float> w(workspace, B, maxT, maxU);
    return launch_finish_costs(w.llf, w.llb, costs, B, nullptr, s);
}

// argument checks of rnnt_entrypoint.cpp:49-60, shared by the loss-op entries (out: the costs, or the 16-bit gradients)
bool loss_args_ok(const void* acts, const int* labels, const int* ylen, const int* xlen, int V, int B, const void* out,
                  const void* workspace, const rnntOptions& o) {
    return acts && labels && ylen && xlen && out && workspace && V > 0 && B > 0 && o.maxT > 0 && o.maxU > 0;
}

// argument checks of the 16-bit entries (those of rnntb200_loss_device, plus the logit type, the blank index and the
// wavefront's maxU bound, so that the backward rejects what its forward would have)
bool loss16_args_ok(const void* acts, int logit_type, const int* labels, const int* ylen, const int* xlen, int V, int B,
                    const void* out, const void* workspace, const rnntOptions& o) {
    return loss_args_ok(acts, labels, ylen, xlen, V, B, out, workspace, o) && o.maxU <= 1024 && o.blank_label >= 0 &&
           o.blank_label < V && (logit_type == RNNTB200_LOGITS_F16 || logit_type == RNNTB200_LOGITS_BF16);
}

// f(logits, gradients) with the pointers typed by the 16-bit logit type (loss16_args_ok has checked it)
template <typename F>
rnntStatus_t with_logits16(int logit_type, const void* acts, void* grads, F&& f) {
    if (logit_type == RNNTB200_LOGITS_F16) return f(static_cast<const __half*>(acts), static_cast<__half*>(grads));
    return f(static_cast<const __nv_bfloat16*>(acts), static_cast<__nv_bfloat16*>(grads));
}

// FastEmit's lambda: finite and >= 0 (NaN fails both comparisons)
inline bool fastemit_ok(float lambda) { return lambda >= 0.f && lambda <= FLT_MAX; }

template <typename T>
rnntStatus_t compute_impl(const T* acts, T* grads, const int* labels, const int* ylen, const int* xlen, int V, int B,
                          T* costs_host, void* workspace, rnntOptions opt) {
    if (!loss_args_ok(acts, labels, ylen, xlen, V, B, costs_host, workspace, opt)) return RNNT_STATUS_INVALID_VALUE;
    if (opt.loc == RNNT_CPU) {
        fprintf(stderr, "rnnt_b200: RNNT_CPU requested but this library has no CPU path (no fallback by design)\n");
        return RNNT_STATUS_EXECUTION_FAILED;
    }
    if (opt.loc != RNNT_GPU) return RNNT_STATUS_INVALID_VALUE;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(opt.stream);
    const bool vec = vec_ok<T>(acts, grads, V);
    rnntStatus_t st = loss_planes<T, T>(acts, vec, labels, ylen, xlen, V, B, opt.maxT, opt.maxU, opt.blank_label, workspace, s);
    if (!st && grads)
        st = loss_grads<T, T>(acts, grads, vec, labels, ylen, xlen, nullptr, V, B, opt.maxT, opt.maxU, opt.blank_label,
                              workspace, s, 0.f);
    if (st) return st;
    // costs to HOST + sync + negate, as gpu_rnnt.h:209-213; llBackward comes along for the guard of cpu_rnnt.h:166-170
    LossWs<T> w(workspace, B, opt.maxT, opt.maxU);
    std::vector<T> llb((size_t)B);
    if (cudaMemcpyAsync(costs_host, w.llf, sizeof(T) * B, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
        cudaMemcpyAsync(llb.data(), w.llb, sizeof(T) * B, cudaMemcpyDeviceToHost, s) != cudaSuccess)
        return RNNT_STATUS_MEMOPS_FAILED;
    if (cudaStreamSynchronize(s) != cudaSuccess) return RNNT_STATUS_EXECUTION_FAILED;
    for (int i = 0; i < B; ++i) {
        const double diff = fabs((double)costs_host[i] - (double)llb[i]);
        if (diff > 0.1) printf("WARNING: Forward backward likelihood mismatch %f\n", diff);   // cpu_rnnt.h:167-170
        costs_host[i] = -costs_host[i];
    }
    return RNNT_STATUS_SUCCESS;
}

// ------------------------------------------------------------------------------------------
// joint path workspace
// ------------------------------------------------------------------------------------------
struct JointWs {
    LossWs<float> loss;
    char* scratch;     // path-specific
    size_t scratch_bytes;
    long long chunk_rows;  // exact path
    size_t total;
    JointWs(const rnntb200JointDesc& d, void* base) : loss(base, d.B, d.maxT, d.maxU) {
        const size_t N = (size_t)d.B * d.maxT * d.maxU;
        size_t off = align_up(loss.bytes, 256);
        scratch = static_cast<char*>(base) + off;
        if (d.precision == RNNTB200_FP32_EXACT) {
            const size_t per_row = (size_t)(2 * d.H + d.V) * sizeof(float);
            size_t ch = ((size_t)1 << 30) / per_row;
            if (ch < 256) ch = 256;
            if (ch > N) ch = N;
            chunk_rows = (long long)ch;
            scratch_bytes = ch * per_row;
        } else {
            chunk_rows = 0;
#ifndef RNNTB200_NO_TC
            scratch_bytes = rb::tc_scratch_bytes(d);
#else
            scratch_bytes = 0;
#endif
        }
        total = off + align_up(scratch_bytes, 256);
    }
};

bool desc_ok(const rnntb200JointDesc* d) {
    return d && d->B > 0 && d->maxT > 0 && d->maxU > 0 && d->H > 0 && d->V > 0 && d->blank_label >= 0 &&
           d->blank_label < d->V && (d->precision == RNNTB200_FP32_EXACT || d->precision == RNNTB200_BF16_TC) &&
           d->maxU <= 1024;
}

inline unsigned ew_blocks(long long total) {
    long long b = (total + 255) / 256;
    return (unsigned)(b > 132 * 32 ? 132 * 32 : (b < 1 ? 1 : b));
}

// C[M,N] (+)= A.B with generic strides; picks the 128x128 float4 kernel when alignment allows.  The row tiles go in
// gridDim.y, which holds at most 65535 of them: a taller product runs as one launch per 65535 row tiles, each on the
// rows m0 .. m0+mc of A and C (A + m0*sAm, C + m0*ldc; 128-row steps keep the fast kernel's 16-byte alignment).
template <bool AK, bool BN_>
void launch_sgemm(const float* A, const float* Bm, float* C, const float* bias, int M, int N, int K, long long sAm,
                  long long sAk, long long sBk, long long sBn, long long ldc, int accumulate, cudaStream_t s) {
    auto al16 = [](const void* p) { return ((uintptr_t)p % 16) == 0; };
    const bool a_ok = AK ? (K % 4 == 0 && sAm % 4 == 0) : (M % 4 == 0 && sAk % 4 == 0);
    const bool b_ok = BN_ ? (N % 4 == 0 && sBk % 4 == 0) : (K % 4 == 0 && sBn % 4 == 0);
    const bool fast = a_ok && b_ok && N % 4 == 0 && ldc % 4 == 0 && al16(A) && al16(Bm) && al16(C) && (!bias || al16(bias));
    const long long mstep = 65535LL * (fast ? 128 : 64);
    for (long long m0 = 0; m0 < M; m0 += mstep) {
        const int mc = (int)(M - m0 < mstep ? M - m0 : mstep);
        const float* Am = A + m0 * sAm;
        float* Cm = C + m0 * ldc;
        if (fast) {
            // few output tiles but a long K (dW = Z^T.dL): split K over blockIdx.z so the grid fills the 132 SMs;
            // only for accumulating calls, whose output already holds valid data to atomically add into
            int splits = 1;
            const int tiles = ((N + 127) / 128) * ((mc + 127) / 128);
            if (accumulate && tiles < 132 && K >= 4096) {
                splits = (132 * 4 + tiles - 1) / tiles;
                if (splits > K / 512) splits = K / 512;
                if (splits < 1) splits = 1;
            }
            dim3 grid((N + 127) / 128, (unsigned)((mc + 127) / 128), splits);
            rb::sgemm128_kernel<AK, BN_><<<grid, 256, 0, s>>>(Am, Bm, Cm, bias, mc, N, K, sAm, sAk, sBk, sBn, ldc, accumulate);
        } else {
            dim3 grid((N + 63) / 64, (unsigned)((mc + 63) / 64));
            rb::sgemm_kernel<AK, BN_><<<grid, 256, 0, s>>>(Am, Bm, Cm, bias, mc, N, K, sAm, sAk, sBk, sBn, ldc, accumulate);
        }
        RB_LAUNCHED(1);
    }
}
// Rows r0 .. r0+rows of the exact path's projection: Z = tanh(enc + pred) (model.py:158-163), then L = Z.W + b
void exact_project(const rnntb200JointDesc& d, const float* enc, const float* pred, const float* W, const float* bias,
                   long long r0, long long rows, float* Z, float* L, cudaStream_t s) {
    rb::zgen_kernel<<<ew_blocks(rows * d.H), 256, 0, s>>>(enc, pred, Z, r0, rows, d.maxT, d.maxU, d.H);
    RB_LAUNCHED(1);
    rb::ScopedTimer tm("sgemm L=Z.W+b", s);
    launch_sgemm<true, true>(Z, W, L, bias, (int)rows, d.V, d.H, d.H, 1, d.V, 1, d.V, 0, s);
}

rnntStatus_t exact_forward(const rnntb200JointDesc& d, const JointWs& ws, const float* enc, const float* pred,
                           const float* W, const float* bias, const int* labels, const int* ylen, const int* xlen,
                           cudaStream_t s, const rb::Windows& win) {
    const long long N = (long long)d.B * d.maxT * d.maxU, SK = skew_plane(d.maxT, d.maxU);
    float* Z = reinterpret_cast<float*>(ws.scratch);
    float* L = Z + ws.chunk_rows * d.H;
    for (long long r0 = 0; r0 < N; r0 += ws.chunk_rows) {
        const long long rows = (N - r0 < ws.chunk_rows) ? N - r0 : ws.chunk_rows;
        exact_project(d, enc, pred, W, bias, r0, rows, Z, L, s);
        rb::lse_gather_kernel<float><<<(unsigned)((rows * 32 + 255) / 256), 256, 0, s>>>(
            L, r0, rows, d.V, xlen, ylen, labels, d.maxT, d.maxU, SK, d.blank_label, ws.loss.lse, ws.loss.lpb,
            ws.loss.lpl, win);
        RB_LAUNCHED(1);
        if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    }
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t exact_backward(const rnntb200JointDesc& d, const JointWs& ws, const float* enc, const float* pred,
                            const float* W, const float* bias, const int* labels, const int* ylen, const int* xlen,
                            const float* grad_costs, float* d_enc, float* d_pred, float* dW, float* db,
                            cudaStream_t s, float fastemit_lambda, const rb::Windows& win) {
    const long long N = (long long)d.B * d.maxT * d.maxU, SK = skew_plane(d.maxT, d.maxU);
    float* Z = reinterpret_cast<float*>(ws.scratch);
    float* L = Z + ws.chunk_rows * d.H;
    float* dZ = L + ws.chunk_rows * d.V;
    if (cudaMemsetAsync(d_enc, 0, sizeof(float) * (size_t)d.B * d.maxT * d.H, s) != cudaSuccess ||
        cudaMemsetAsync(d_pred, 0, sizeof(float) * (size_t)d.B * d.maxU * d.H, s) != cudaSuccess ||
        cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)d.H * d.V, s) != cudaSuccess ||
        cudaMemsetAsync(db, 0, sizeof(float) * (size_t)d.V, s) != cudaSuccess)
        return RNNT_STATUS_MEMOPS_FAILED;
    for (long long r0 = 0; r0 < N; r0 += ws.chunk_rows) {
        const long long rows = (N - r0 < ws.chunk_rows) ? N - r0 : ws.chunk_rows;
        exact_project(d, enc, pred, W, bias, r0, rows, Z, L, s);
        // dlogits in place (gpu_rnnt_kernel.h:143-179 formula, times the upstream per-utterance gradient)
        rb::rnnt_grad_kernel<float><<<(unsigned)((rows * 32 + 255) / 256), 256, 0, s>>>(
            L, L, r0, rows, d.V, xlen, ylen, labels, d.maxT, d.maxU, SK, d.blank_label, ws.loss.lse, ws.loss.alphas,
            ws.loss.betas, ws.loss.llf, grad_costs, fastemit_lambda, win);
        // dZ = dL . W^T      (rows x V) . (V x H):  B(k=v, n=h) = W[h*V + v]
        {
            rb::ScopedTimer tm("sgemm dZ=dL.W^T", s);
            launch_sgemm<true, false>(L, W, dZ, nullptr, (int)rows, d.H, d.V, d.V, 1, 1, d.V, d.H, 0, s);
        }
        rb::dz_reduce_kernel<<<ew_blocks(rows * d.H), 256, 0, s>>>(dZ, Z, r0, rows, d.maxT, d.maxU, d.H, d_enc,
                                                                   d_pred);
        // dW += Z^T . dL     (H x rows) . (rows x V):  A(m=h, k=r) = Z[r*H + h]
        {
            rb::ScopedTimer tm("sgemm dW+=Z^T.dL", s);
            launch_sgemm<false, true>(Z, L, dW, nullptr, d.H, d.V, (int)rows, 1, d.H, d.V, 1, d.V, 1, s);
        }
        {
            long long gy = (rows + 255) / 256;
            if (gy > 512) gy = 512;
            rb::colsum_kernel<<<dim3((d.V + 31) / 32, (unsigned)gy), 256, 0, s>>>(L, rows, d.V, db);
        }
        RB_LAUNCHED(4);
        if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    }
    return RNNT_STATUS_SUCCESS;
}

#ifdef RNNTB200_NO_TC
inline rnntStatus_t tc_missing() {
    fprintf(stderr, "rnnt_b200: built without the tensor-core path\n");
    return RNNT_STATUS_EXECUTION_FAILED;
}
#endif

// The joint forward of the loss and alignment entries: projection (exact or tensor-core), alpha/beta, costs.  *overflow:
// the broken-valid_tile_bound word finish_costs reads (nullptr: none).  A keeping forward has just ranked the tiles, so
// its word is fresh; one that keeps nothing counts them only for the alignment (check_bound).
rnntStatus_t joint_forward(const rnntb200JointDesc& d, const JointWs& ws, const float* enc, const float* pred,
                           const float* W, const float* bias, const int* labels, const int* ylen, const int* xlen,
                           float* costs, bool check_bound, const int** overflow, cudaStream_t s,
                           const rb::Windows& win = no_windows) {
    *overflow = nullptr;
    rnntStatus_t st;
    if (d.precision == RNNTB200_FP32_EXACT) {
        st = exact_forward(d, ws, enc, pred, W, bias, labels, ylen, xlen, s, win);
    } else {
#ifndef RNNTB200_NO_TC
        unsigned nl = 0;
        st = rb::tc_forward(d, ws.scratch, enc, pred, W, bias, labels, ylen, xlen, ws.loss.lse, ws.loss.lpb, ws.loss.lpl,
                            s, &nl, win);
        if (!st) {
            const rb::TcScratch sc = rb::tc_scratch_layout(d, ws.scratch);
            if (check_bound) *overflow = rb::tc_check_tile_bound(d, ws.scratch, ylen, xlen, s, &nl);
            else if (rb::tc_keep(d, sc)) *overflow = sc.count + 1;
        }
        RB_LAUNCHED(nl);
#else
        st = tc_missing();
#endif
    }
    if (st) return st;
    st = launch_alpha_beta(ws.loss, xlen, ylen, d.B, d.maxT, d.maxU, s, win);
    if (st) return st;
    return launch_finish_costs(ws.loss.llf, ws.loss.llb, costs, d.B, *overflow, s);
}

// argument checks shared by the joint entries that run the loss (forward, backward, alignment)
bool joint_loss_args_ok(const rnntb200JointDesc* d, const float* enc, const float* pred, const float* W,
                        const float* bias, const int* labels, const int* ylen, const int* xlen, const void* workspace) {
    return desc_ok(d) && enc && pred && W && bias && labels && ylen && xlen && workspace;
}

// ------------------------------------------------------------------------------------------
// simple (trivial-joiner) loss of pruned RNN-T (csrc/simple_joiner.cuh)
// ------------------------------------------------------------------------------------------
// Workspace: the loss op's planes (LossWs), the row maxima, Ea / El, the normaliser plane (forward), the G plane
// (backward), the underflow flags and the two band planes of the windows call.  Each call writes only its own parts, so
// the backward and the windows call leave what the forward wrote unchanged.  Ea / El come last: the windows call has no V
// and locates everything else with V = 0.
struct SimpleWs {
    LossWs<float> loss;
    float *ma, *ml, *nrm, *G, *Ea, *El;
    unsigned char* flag;
    int *s_raw, *s_band;
    size_t total;
    SimpleWs(void* base, int B, int maxT, int maxU, int V) : loss(base, B, maxT, maxU) {
        const size_t NT = (size_t)B * maxT, NU = (size_t)B * maxU, N = NT * maxU;
        char* p = static_cast<char*>(base);
        size_t off = align_up(loss.bytes, 256);
        auto take = [&](size_t bytes) { char* q = p + off; off += align_up(bytes, 256); return q; };
        ma = reinterpret_cast<float*>(take(NT * 4));
        ml = reinterpret_cast<float*>(take(NU * 4));
        nrm = reinterpret_cast<float*>(take(N * 4));
        G = reinterpret_cast<float*>(take(N * 4));
        flag = reinterpret_cast<unsigned char*>(take(N));
        s_raw = reinterpret_cast<int*>(take(NT * 4));
        s_band = reinterpret_cast<int*>(take(NT * 4));
        Ea = reinterpret_cast<float*>(take(NT * V * 4));
        El = reinterpret_cast<float*>(take(NU * V * 4));
        total = off;
    }
};

bool simple_args_ok(const float* am, const float* lm, const int* labels, const int* ylen, const int* xlen, int V, int B,
                    const void* workspace, const rnntOptions& o) {
    return am && lm && labels && ylen && xlen && workspace && V > 0 && B > 0 && o.maxT > 0 && o.maxU > 0 &&
           o.maxU <= 1024 && o.blank_label >= 0 && o.blank_label < V;
}

// C[b] (M x N) = A[b] . B[b] (EPI 0) or X[b] (.) (A[b] . B[b]) (EPI 1), one launch per 65535 batches
template <bool AK, bool BN, int EPI>
void launch_bgemm(const float* A, const float* Bm, float* C, const float* X, int M, int N, int K, long long sA, long long sB,
                  long long ldc, long long bA, long long bB, long long bC, int batches, cudaStream_t s) {
    for (int b0 = 0; b0 < batches; b0 += 65535) {
        const int nb = min(65535, batches - b0);
        dim3 grid((N + 127) / 128, (M + 127) / 128, nb);
        rb::bgemm_kernel<AK, BN, EPI><<<grid, 256, 0, s>>>(A + b0 * bA, Bm + b0 * bB, C + b0 * bC, EPI ? X + b0 * bC : nullptr,
                                                           M, N, K, sA, sB, ldc, bA, bB, bC);
        RB_LAUNCHED(1);
    }
}

}  // namespace

extern "C" {

int get_warprnnt_version() { return 1; }

const char* rnntGetStatusString(rnntStatus_t status) {
    switch (status) {
        case RNNT_STATUS_SUCCESS: return "no error";
        case RNNT_STATUS_MEMOPS_FAILED: return "cuda memcpy or memset failed";
        case RNNT_STATUS_INVALID_VALUE: return "invalid value";
        case RNNT_STATUS_EXECUTION_FAILED: return "execution failed";
        case RNNT_STATUS_UNKNOWN_ERROR:
        default: return "unknown error";
    }
}

rnntStatus_t get_workspace_size(int maxT, int maxU, int minibatch, bool gpu, size_t* size_bytes, size_t dtype_size) {
    if (minibatch <= 0 || maxT <= 0 || maxU <= 0 || !size_bytes) return RNNT_STATUS_INVALID_VALUE;
    if (!gpu) {  // reference CPU figure, rnnt_entrypoint.cpp:109-118 (informational only)
        *size_bytes = dtype_size * (size_t)maxT * maxU * 4 * (size_t)minibatch;
        return RNNT_STATUS_SUCCESS;
    }
    const size_t SK = (size_t)skew_plane(maxT, maxU);
    *size_bytes = (size_t)minibatch * (4 * SK + (size_t)maxT * maxU + 2) * dtype_size;
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t compute_rnnt_loss(const float* const activations, float* gradients, const int* const flat_labels,
                               const int* const label_lengths, const int* const input_lengths, int alphabet_size,
                               int minibatch, float* costs, void* workspace, rnntOptions options) {
    return compute_impl<float>(activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size,
                               minibatch, costs, workspace, options);
}

rnntStatus_t compute_rnnt_loss_fp64(const double* const activations, double* gradients,
                                    const int* const flat_labels, const int* const label_lengths,
                                    const int* const input_lengths, int alphabet_size, int minibatch,
                                    double* costs, void* workspace, rnntOptions options) {
    return compute_impl<double>(activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size,
                                minibatch, costs, workspace, options);
}

rnntStatus_t rnntb200_loss_device(const float* activations, float* gradients, const int* flat_labels,
                                  const int* label_lengths, const int* input_lengths, const float* grad_scale,
                                  int alphabet_size, int minibatch, float* costs_device, void* workspace,
                                  rnntOptions options) {
    return rnntb200_loss_device_fastemit(activations, gradients, flat_labels, label_lengths, input_lengths, grad_scale,
                                         alphabet_size, minibatch, costs_device, workspace, options, 0.f);
}

rnntStatus_t rnntb200_loss_device_fastemit(const float* activations, float* gradients, const int* flat_labels,
                                           const int* label_lengths, const int* input_lengths, const float* grad_scale,
                                           int alphabet_size, int minibatch, float* costs_device, void* workspace,
                                           rnntOptions options, float fastemit_lambda) {
    return rnntb200_loss_device_windowed(activations, gradients, flat_labels, label_lengths, input_lengths, grad_scale,
                                         nullptr, nullptr, alphabet_size, minibatch, costs_device, workspace, options,
                                         fastemit_lambda);
}

rnntStatus_t rnntb200_loss_device_windowed(const float* activations, float* gradients, const int* flat_labels,
                                           const int* label_lengths, const int* input_lengths, const float* grad_scale,
                                           const int* t_lo, const int* t_hi, int alphabet_size, int minibatch,
                                           float* costs_device, void* workspace, rnntOptions options,
                                           float fastemit_lambda) {
    if (!loss_args_ok(activations, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch, costs_device,
                      workspace, options) || !fastemit_ok(fastemit_lambda) || !windows_ok(t_lo, t_hi))
        return RNNT_STATUS_INVALID_VALUE;
    const rb::Windows win{t_lo, t_hi};
    cudaStream_t s = reinterpret_cast<cudaStream_t>(options.stream);
    const int V = alphabet_size, B = minibatch, T = options.maxT, U = options.maxU, blank = options.blank_label;
    const bool vec = vec_ok<float>(activations, gradients, V);
    rnntStatus_t st = loss_forward(activations, vec, flat_labels, label_lengths, input_lengths, V, B, T, U, blank,
                                   costs_device, workspace, s, win);
    if (st || !gradients) return st;
    return loss_grads<float, float>(activations, gradients, vec, flat_labels, label_lengths, input_lengths, grad_scale, V,
                                    B, T, U, blank, workspace, s, fastemit_lambda, win);
}

rnntStatus_t rnntb200_loss16_forward(const void* activations, int logit_type, const int* flat_labels,
                                     const int* label_lengths, const int* input_lengths, int alphabet_size, int minibatch,
                                     float* costs_device, void* workspace, rnntOptions options) {
    return rnntb200_loss16_forward_windowed(activations, logit_type, flat_labels, label_lengths, input_lengths, nullptr,
                                            nullptr, alphabet_size, minibatch, costs_device, workspace, options);
}

rnntStatus_t rnntb200_loss16_forward_windowed(const void* activations, int logit_type, const int* flat_labels,
                                              const int* label_lengths, const int* input_lengths, const int* t_lo,
                                              const int* t_hi, int alphabet_size, int minibatch, float* costs_device,
                                              void* workspace, rnntOptions options) {
    if (!loss16_args_ok(activations, logit_type, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                        costs_device, workspace, options) || !windows_ok(t_lo, t_hi))
        return RNNT_STATUS_INVALID_VALUE;
    const rb::Windows win{t_lo, t_hi};
    cudaStream_t s = reinterpret_cast<cudaStream_t>(options.stream);
    const int V = alphabet_size, B = minibatch, T = options.maxT, U = options.maxU, blank = options.blank_label;
    return with_logits16(logit_type, activations, nullptr, [&](auto x, auto g) {
        return loss_forward(x, vec_ok<float>(x, g, V), flat_labels, label_lengths, input_lengths, V, B, T, U, blank,
                            costs_device, workspace, s, win);
    });
}

rnntStatus_t rnntb200_loss16_backward(const void* activations, int logit_type, const int* flat_labels,
                                      const int* label_lengths, const int* input_lengths, const float* grad_costs,
                                      int alphabet_size, int minibatch, void* gradients, const void* workspace,
                                      rnntOptions options) {
    return rnntb200_loss16_backward_fastemit(activations, logit_type, flat_labels, label_lengths, input_lengths, grad_costs,
                                             alphabet_size, minibatch, gradients, workspace, options, 0.f);
}

rnntStatus_t rnntb200_loss16_backward_fastemit(const void* activations, int logit_type, const int* flat_labels,
                                               const int* label_lengths, const int* input_lengths, const float* grad_costs,
                                               int alphabet_size, int minibatch, void* gradients, const void* workspace,
                                               rnntOptions options, float fastemit_lambda) {
    return rnntb200_loss16_backward_windowed(activations, logit_type, flat_labels, label_lengths, input_lengths, nullptr,
                                             nullptr, grad_costs, alphabet_size, minibatch, gradients, workspace, options,
                                             fastemit_lambda);
}

rnntStatus_t rnntb200_loss16_backward_windowed(const void* activations, int logit_type, const int* flat_labels,
                                               const int* label_lengths, const int* input_lengths, const int* t_lo,
                                               const int* t_hi, const float* grad_costs, int alphabet_size, int minibatch,
                                               void* gradients, const void* workspace, rnntOptions options,
                                               float fastemit_lambda) {
    if (!loss16_args_ok(activations, logit_type, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                        gradients, workspace, options) || !fastemit_ok(fastemit_lambda) || !windows_ok(t_lo, t_hi))
        return RNNT_STATUS_INVALID_VALUE;
    const rb::Windows win{t_lo, t_hi};
    cudaStream_t s = reinterpret_cast<cudaStream_t>(options.stream);
    const int V = alphabet_size, B = minibatch, T = options.maxT, U = options.maxU, blank = options.blank_label;
    void* ws = const_cast<void*>(workspace);      // read only: LossWs just carves the planes out of it
    return with_logits16(logit_type, activations, gradients, [&](auto x, auto g) {
        return loss_grads<float>(x, g, vec_ok<float>(x, g, V), flat_labels, label_lengths, input_lengths, grad_costs, V, B,
                                 T, U, blank, ws, s, fastemit_lambda, win);
    });
}

rnntStatus_t rnntb200_joint_workspace_size(const rnntb200JointDesc* desc, size_t* size_bytes) {
    if (!desc_ok(desc) || !size_bytes) return RNNT_STATUS_INVALID_VALUE;
    JointWs ws(*desc, nullptr);
    *size_bytes = ws.total;
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t rnntb200_joint_loss_forward(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                         const float* W, const float* bias, const int* labels,
                                         const int* label_lengths, const int* input_lengths, float* costs,
                                         void* workspace) {
    return rnntb200_joint_loss_forward_windowed(desc, enc, pred, W, bias, labels, label_lengths, input_lengths, nullptr,
                                                nullptr, costs, workspace);
}

rnntStatus_t rnntb200_joint_loss_forward_windowed(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                                  const float* W, const float* bias, const int* labels,
                                                  const int* label_lengths, const int* input_lengths, const int* t_lo,
                                                  const int* t_hi, float* costs, void* workspace) {
    if (!joint_loss_args_ok(desc, enc, pred, W, bias, labels, label_lengths, input_lengths, workspace) || !costs ||
        !windows_ok(t_lo, t_hi))
        return RNNT_STATUS_INVALID_VALUE;
    const int* overflow;
    return joint_forward(*desc, JointWs(*desc, workspace), enc, pred, W, bias, labels, label_lengths, input_lengths, costs,
                         false, &overflow, reinterpret_cast<cudaStream_t>(desc->stream), rb::Windows{t_lo, t_hi});
}

rnntStatus_t rnntb200_joint_loss_backward(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                          const float* W, const float* bias, const int* labels,
                                          const int* label_lengths, const int* input_lengths,
                                          const float* grad_costs, float* d_enc, float* d_pred, float* dW,
                                          float* db, void* workspace) {
    return rnntb200_joint_loss_backward_fastemit(desc, enc, pred, W, bias, labels, label_lengths, input_lengths, grad_costs,
                                                 d_enc, d_pred, dW, db, workspace, 0.f);
}

rnntStatus_t rnntb200_joint_loss_backward_fastemit(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                                   const float* W, const float* bias, const int* labels,
                                                   const int* label_lengths, const int* input_lengths,
                                                   const float* grad_costs, float* d_enc, float* d_pred, float* dW,
                                                   float* db, void* workspace, float fastemit_lambda) {
    return rnntb200_joint_loss_backward_windowed(desc, enc, pred, W, bias, labels, label_lengths, input_lengths, nullptr,
                                                 nullptr, grad_costs, d_enc, d_pred, dW, db, workspace, fastemit_lambda);
}

rnntStatus_t rnntb200_joint_loss_backward_windowed(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                                   const float* W, const float* bias, const int* labels,
                                                   const int* label_lengths, const int* input_lengths, const int* t_lo,
                                                   const int* t_hi, const float* grad_costs, float* d_enc, float* d_pred,
                                                   float* dW, float* db, void* workspace, float fastemit_lambda) {
    if (!joint_loss_args_ok(desc, enc, pred, W, bias, labels, label_lengths, input_lengths, workspace) || !grad_costs ||
        !d_enc || !d_pred || !dW || !db || !fastemit_ok(fastemit_lambda) || !windows_ok(t_lo, t_hi))
        return RNNT_STATUS_INVALID_VALUE;
    const rb::Windows win{t_lo, t_hi};
    const rnntb200JointDesc& d = *desc;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(d.stream);
    JointWs ws(d, workspace);
    if (d.precision == RNNTB200_FP32_EXACT)
        return exact_backward(d, ws, enc, pred, W, bias, labels, label_lengths, input_lengths, grad_costs, d_enc,
                              d_pred, dW, db, s, fastemit_lambda, win);
#ifndef RNNTB200_NO_TC
    unsigned nl = 0;
    const rb::LossPlanes lp{ws.loss.lse, ws.loss.lpb, ws.loss.lpl, ws.loss.alphas, ws.loss.betas, ws.loss.llf};
    rnntStatus_t st = rb::tc_backward(d, ws.scratch, enc, pred, bias, labels, label_lengths, input_lengths, lp, grad_costs,
                                      d_enc, d_pred, dW, db, s, &nl, fastemit_lambda, win);
    RB_LAUNCHED(nl);
    return st;
#else
    return tc_missing();
#endif
}

rnntStatus_t rnntb200_align_device(const float* activations, const int* flat_labels, const int* label_lengths,
                                   const int* input_lengths, int alphabet_size, int minibatch, float* costs_device,
                                   float* best_logp, int* label_frames, void* workspace, rnntOptions options) {
    if (!align_args_ok(best_logp, label_frames, options.maxU) || options.maxU > 1024 || options.blank_label < 0 ||
        options.blank_label >= alphabet_size)
        return RNNT_STATUS_INVALID_VALUE;
    rnntStatus_t st = rnntb200_loss_device(activations, nullptr, flat_labels, label_lengths, input_lengths, nullptr,
                                           alphabet_size, minibatch, costs_device, workspace, options);
    if (st) return st;
    LossWs<float> w(workspace, minibatch, options.maxT, options.maxU);
    return launch_align(w, input_lengths, label_lengths, minibatch, options.maxT, options.maxU, nullptr, best_logp,
                        label_frames, reinterpret_cast<cudaStream_t>(options.stream));
}

rnntStatus_t rnntb200_align16(const void* activations, int logit_type, const int* flat_labels, const int* label_lengths,
                              const int* input_lengths, int alphabet_size, int minibatch, float* costs_device,
                              float* best_logp, int* label_frames, void* workspace, rnntOptions options) {
    if (!align_args_ok(best_logp, label_frames, options.maxU)) return RNNT_STATUS_INVALID_VALUE;
    rnntStatus_t st = rnntb200_loss16_forward(activations, logit_type, flat_labels, label_lengths, input_lengths,
                                              alphabet_size, minibatch, costs_device, workspace, options);
    if (st) return st;
    LossWs<float> w(workspace, minibatch, options.maxT, options.maxU);
    return launch_align(w, input_lengths, label_lengths, minibatch, options.maxT, options.maxU, nullptr, best_logp,
                        label_frames, reinterpret_cast<cudaStream_t>(options.stream));
}

rnntStatus_t rnntb200_joint_align(const rnntb200JointDesc* desc, const float* enc, const float* pred, const float* W,
                                  const float* bias, const int* labels, const int* label_lengths,
                                  const int* input_lengths, float* costs, float* best_logp, int* label_frames,
                                  void* workspace) {
    if (!joint_loss_args_ok(desc, enc, pred, W, bias, labels, label_lengths, input_lengths, workspace) || !costs ||
        !align_args_ok(best_logp, label_frames, desc->maxU))
        return RNNT_STATUS_INVALID_VALUE;
    rnntb200JointDesc d = *desc;
    d.keep_activations = 0;                 // no backward follows: nothing beyond the loss planes is kept
    cudaStream_t s = reinterpret_cast<cudaStream_t>(d.stream);
    JointWs ws(d, workspace);
    const int* overflow;
    rnntStatus_t st = joint_forward(d, ws, enc, pred, W, bias, labels, label_lengths, input_lengths, costs, true, &overflow, s);
    if (st) return st;
    return launch_align(ws.loss, input_lengths, label_lengths, d.B, d.maxT, d.maxU, overflow, best_logp, label_frames, s);
}

rnntStatus_t rnntb200_joint_logits(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                   const float* W, const float* bias, float* logits, void* workspace) {
    if (!desc_ok(desc) || !enc || !pred || !W || !bias || !logits || !workspace) return RNNT_STATUS_INVALID_VALUE;
    rnntb200JointDesc d = *desc;
    d.precision = RNNTB200_FP32_EXACT;  // the materialising entry is the fp32 literal of model.py:158-166
    cudaStream_t s = reinterpret_cast<cudaStream_t>(d.stream);
    JointWs ws(d, workspace);
    const long long N = (long long)d.B * d.maxT * d.maxU;
    for (long long r0 = 0; r0 < N; r0 += ws.chunk_rows) {
        const long long rows = (N - r0 < ws.chunk_rows) ? N - r0 : ws.chunk_rows;
        exact_project(d, enc, pred, W, bias, r0, rows, reinterpret_cast<float*>(ws.scratch), logits + r0 * d.V, s);
        if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    }
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t rnntb200_joint_step(const float* f, long long ldf, const float* g, long long ldg, const float* K1,
                                 const float* b1, const float* K2, const float* b2, int B, int P, int H, int V,
                                 float* logits, int* best, float* best_logp, CUstream stream) {
    if (!f || !g || !K2 || B <= 0 || P <= 0 || H <= 0 || V <= 0 || (!logits && !best && !best_logp)) return RNNT_STATUS_INVALID_VALUE;
    if (!K1 && P != H) return RNNT_STATUS_INVALID_VALUE;
    if (P > rb::STEP_MAX_DIM || H > rb::STEP_CLUSTER * rb::STEP_THREADS) {
        fprintf(stderr, "rnnt_b200: rnntb200_joint_step supports P <= %d, H <= %d\n", rb::STEP_MAX_DIM, rb::STEP_CLUSTER * rb::STEP_THREADS);
        return RNNT_STATUS_INVALID_VALUE;
    }
    if (V > rb::joint_step_max_v(P, H)) {     // each CTA keeps its eighth of the logits in shared memory
        fprintf(stderr, "rnnt_b200: rnntb200_joint_step supports V <= %d at P = %d, H = %d\n", rb::joint_step_max_v(P, H), P, H);
        return RNNT_STATUS_INVALID_VALUE;
    }
    rb::StepParams p{f, g, ldf, ldg, K1, b1, K2, b2, B, P, H, V, logits, best, best_logp};
    const size_t smem = rb::joint_step_smem(P, H, V);
    if (smem > rb::STEP_SMEM_DEFAULT &&
        !rb::tc_smem_optin(reinterpret_cast<const void*>(rb::joint_step_kernel), rb::STEP_SMEM_MAX))
        return RNNT_STATUS_EXECUTION_FAILED;
    rb::joint_step_kernel<<<B * rb::STEP_CLUSTER, rb::STEP_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    RB_LAUNCHED(1);
    return check_launch();
}

// Dense-1 of the joint, hoisted in front of the broadcast add (SURVEY 8 a2 / f1): three strided products of the library's
// fp32 FMA GEMM kernel and one column sum.
rnntStatus_t rnntb200_dense1_forward(const float* X, long long rows, int P, const float* K1, const float* b1, int H,
                                     float* out, CUstream stream) {
    if (!X || !K1 || !out || rows <= 0 || rows > INT_MAX || P <= 0 || H <= 0) return RNNT_STATUS_INVALID_VALUE;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    rb::ScopedTimer tm("dense1 X.K1+b1", s);
    launch_sgemm<true, true>(X, K1, out, b1, (int)rows, H, P, P, 1, H, 1, H, 0, s);
    return check_launch();
}

rnntStatus_t rnntb200_dense1_backward(const float* X, const float* dA, const float* K1, long long rows, int P, int H,
                                      float* dX, float* dK1, float* db1, CUstream stream) {
    if (!dA || rows <= 0 || rows > INT_MAX || P <= 0 || H <= 0 || (dX && !K1) || (dK1 && !X)) return RNNT_STATUS_INVALID_VALUE;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (dX) {       // dX[r,p] = sum_h dA[r,h] K1[p,h]
        rb::ScopedTimer tm("dense1 dX=dA.K1^T", s);
        launch_sgemm<true, false>(dA, K1, dX, nullptr, (int)rows, P, H, H, 1, 1, H, P, 0, s);
    }
    if (dK1) {      // dK1[p,h] += sum_r X[r,p] dA[r,h]
        rb::ScopedTimer tm("dense1 dK1+=X^T.dA", s);
        launch_sgemm<false, true>(X, dA, dK1, nullptr, P, H, (int)rows, 1, P, H, 1, H, 1, s);
    }
    if (db1) {
        rb::ScopedTimer tm("dense1 db1+=colsum(dA)", s);
        rb::colsum_kernel<<<dim3((H + 31) / 32, 1), 256, 0, s>>>(dA, rows, H, db1);      // one row block: deterministic
        RB_LAUNCHED(1);
    }
    return check_launch();
}

rnntStatus_t rnntb200_simple_workspace_size(int B, int maxT, int maxU, int V, size_t* size_bytes) {
    if (B <= 0 || maxT <= 0 || maxU <= 0 || maxU > 1024 || V <= 0 || !size_bytes) return RNNT_STATUS_INVALID_VALUE;
    *size_bytes = SimpleWs(nullptr, B, maxT, maxU, V).total;
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t rnntb200_simple_loss_forward(const float* am, const float* lm, const int* labels, const int* label_lengths,
                                          const int* input_lengths, int V, int B, float* costs, void* workspace,
                                          rnntOptions options) {
    if (!simple_args_ok(am, lm, labels, label_lengths, input_lengths, V, B, workspace, options) || !costs)
        return RNNT_STATUS_INVALID_VALUE;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(options.stream);
    const int T = options.maxT, U = options.maxU, blank = options.blank_label;
    const SimpleWs w(workspace, B, T, U, V);
    const long long NT = (long long)B * T, NU = (long long)B * U, N = NT * U, SK = skew_plane(T, U);
    {
        rb::ScopedTimer tm("simple_exp_rows_kernel", s);
        rb::simple_exp_rows_kernel<<<(unsigned)((NT * 32 + 255) / 256), 256, 0, s>>>(am, NT, T, V, input_lengths, 0, w.ma, w.Ea);
        rb::simple_exp_rows_kernel<<<(unsigned)((NU * 32 + 255) / 256), 256, 0, s>>>(lm, NU, U, V, label_lengths, 1, w.ml, w.El);
    }
    RB_LAUNCHED(2);
    {   // Nrm[b] = Ea[b] . El[b]^T:  A(t,v) = Ea[t*V + v],  B(v,u) = El[u*V + v]
        rb::ScopedTimer tm("bgemm Nrm=Ea.El^T", s);
        launch_bgemm<true, false, 0>(w.Ea, w.El, w.nrm, nullptr, T, U, V, V, V, U, (long long)T * V, (long long)U * V,
                                     (long long)T * U, B, s);
    }
    {
        rb::ScopedTimer tm("simple_lse_kernel", s);
        rb::simple_lse_kernel<<<(unsigned)((N * 32 + 255) / 256), 256, 0, s>>>(am, lm, w.ma, w.ml, w.nrm, input_lengths,
                                                                            label_lengths, labels, T, U, SK, N, V, blank,
                                                                            w.loss.lse, w.loss.lpb, w.loss.lpl, w.flag);
    }
    RB_LAUNCHED(1);
    if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    if (launch_alpha_beta(w.loss, input_lengths, label_lengths, B, T, U, s)) return RNNT_STATUS_EXECUTION_FAILED;
    return launch_finish_costs(w.loss.llf, w.loss.llb, costs, B, nullptr, s);
}

rnntStatus_t rnntb200_simple_loss_backward(const float* am, const float* lm, const int* labels, const int* label_lengths,
                                           const int* input_lengths, int V, int B, const float* grad_costs, float* d_am,
                                           float* d_lm, void* workspace, rnntOptions options) {
    if (!simple_args_ok(am, lm, labels, label_lengths, input_lengths, V, B, workspace, options) || !d_am || !d_lm)
        return RNNT_STATUS_INVALID_VALUE;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(options.stream);
    const int T = options.maxT, U = options.maxU, blank = options.blank_label;
    const SimpleWs w(workspace, B, T, U, V);
    const LossWs<float>& L = w.loss;
    const long long N = (long long)B * T * U, SK = skew_plane(T, U);
    {
        rb::ScopedTimer tm("simple_g_kernel", s);
        rb::simple_g_kernel<<<(unsigned)((N + 255) / 256), 256, 0, s>>>(w.ma, w.ml, L.lse, L.alphas, L.betas, L.llf, w.flag,
                                                                       grad_costs, input_lengths, label_lengths, T, U, SK,
                                                                       N, w.G);
    }
    RB_LAUNCHED(1);
    {   // d_am[b] = Ea[b] (.) (G[b] . El[b]):  A(t,u) = G[t*U + u],  B(u,v) = El[u*V + v]
        rb::ScopedTimer tm("bgemm d_am=Ea*(G.El)", s);
        launch_bgemm<true, true, 1>(w.G, w.El, d_am, w.Ea, T, V, U, U, V, V, (long long)T * U, (long long)U * V,
                                    (long long)T * V, B, s);
    }
    {   // d_lm[b] = El[b] (.) (G[b]^T . Ea[b]):  A(u,t) = G[t*U + u],  B(t,v) = Ea[t*V + v]
        rb::ScopedTimer tm("bgemm d_lm=El*(G^T.Ea)", s);
        launch_bgemm<false, true, 1>(w.G, w.Ea, d_lm, w.El, U, V, T, U, V, V, (long long)T * U, (long long)T * V,
                                     (long long)U * V, B, s);
    }
    if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    {
        rb::ScopedTimer tm("simple_dam_fix_kernel", s);
        rb::simple_dam_fix_kernel<<<(unsigned)(B * T), rb::SIMPLE_FIX_THREADS, 0, s>>>(
            am, lm, L.lse, L.lpb, L.lpl, L.alphas, L.betas, L.llf, w.flag, grad_costs, input_lengths, label_lengths, labels,
            T, U, SK, V, blank, d_am);
    }
    {
        rb::ScopedTimer tm("simple_dlm_fix_kernel", s);
        rb::simple_dlm_fix_kernel<<<(unsigned)(B * U), rb::SIMPLE_FIX_THREADS, 0, s>>>(
            am, lm, L.lse, L.lpb, L.lpl, L.alphas, L.betas, L.llf, w.flag, grad_costs, input_lengths, label_lengths, labels,
            T, U, SK, V, blank, d_lm);
    }
    RB_LAUNCHED(2);
    return check_launch();
}

rnntStatus_t rnntb200_simple_prune_windows(const int* label_lengths, const int* input_lengths, int B, int s_range,
                                           int* t_lo, int* t_hi, void* workspace, rnntOptions options) {
    if (!label_lengths || !input_lengths || !t_lo || !t_hi || !workspace || B <= 0 || s_range < 2 || options.maxT <= 0 ||
        options.maxU <= 0 || options.maxU > 1024)
        return RNNT_STATUS_INVALID_VALUE;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(options.stream);
    const int T = options.maxT, U = options.maxU;
    const SimpleWs w(workspace, B, T, U, 0);
    const LossWs<float>& L = w.loss;
    {
        rb::ScopedTimer tm("prune_score_kernel", s);
        rb::prune_score_kernel<<<dim3(B, (T + rb::PRUNE_WARPS - 1) / rb::PRUNE_WARPS), rb::PRUNE_WARPS * 32, 0, s>>>(
            L.lpb, L.lpl, L.alphas, L.betas, L.llf, input_lengths, label_lengths, T, U, skew_plane(T, U), s_range, w.s_raw);
    }
    {
        rb::ScopedTimer tm("prune_windows_kernel", s);
        rb::prune_windows_kernel<<<B, rb::PRUNE_THREADS, 0, s>>>(w.s_raw, w.s_band, input_lengths, label_lengths, T, U,
                                                                 s_range, t_lo, t_hi);
    }
    RB_LAUNCHED(2);
    return check_launch();
}

unsigned long long rnntb200_launch_count() { return g_launches.load(); }

void rnntb200_set_timing(int on) { rb::timing_reset(on); }

int rnntb200_get_timing(int index, const char** name, float* ms) {
    auto& v = rb::timing_recs();
    if (index < 0 || index >= (int)v.size() || !name || !ms) return 0;
    *name = v[index].name;
    if (cudaEventElapsedTime(ms, v[index].a, v[index].b) != cudaSuccess) *ms = -1.f;
    return 1;
}

const char* rnntb200_build_info() {
#ifndef RNNTB200_NO_TC
    return "rnnt_b200 0.1 sm_90a wgmma=1";
#else
    return "rnnt_b200 0.1 sm_90a wgmma=0";
#endif
}

}  // extern "C"
