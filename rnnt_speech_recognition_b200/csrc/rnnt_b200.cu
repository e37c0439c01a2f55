// rnnt_b200.cu -- C ABI (include/rnnt_b200.h) and host-side orchestration of the RNN-T loss hot
// path on H100 (sm_90a).  No allocation, no host synchronisation (except the reference-mandated one in
// compute_rnnt_loss), everything stream-ordered on the caller's stream.
#include "../../include/rnnt_b200.h"

#include <atomic>
#include <climits>
#include <cstdio>
#include <cstdint>
#include <cmath>
#include <vector>

#include <cuda_runtime.h>

#include "kernels_simt.cuh"
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
                                    const int* __restrict__ overflow = nullptr) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (overflow && *overflow) { out[i] = __int_as_float(0x7fc00000); return; }   // broken valid_tile_bound promise (tile_compact_kernel reported it)
    out[i] = -llf[i];
    const float diff = fabsf(llf[i] - llb[i]);
    if (diff > 0.1f) printf("WARNING: Forward backward likelihood mismatch %f (utterance %d)\n", diff, i);
}

inline rnntStatus_t check_launch() { return cudaGetLastError() == cudaSuccess ? RNNT_STATUS_SUCCESS : RNNT_STATUS_EXECUTION_FAILED; }

template <typename T>
rnntStatus_t launch_alpha_beta(const LossWs<T>& w, const int* xlen, const int* ylen, int B, int maxT, int maxU,
                               cudaStream_t s) {
    const int threads = (maxU + 31) / 32 * 32;
    constexpr int PF = sizeof(T) == 4 ? 8 : 4;
    rb::ScopedTimer tm("alpha_beta_kernel", s);
    rb::alpha_beta_kernel<T, PF><<<dim3(B, 2), threads, 0, s>>>(w.lpb, w.lpl, w.alphas, w.betas, w.llf, w.llb, xlen,
                                                                ylen, maxU, skew_plane(maxT, maxU));
    RB_LAUNCHED(1);
    return check_launch();
}

// loss op on materialised logits: lse+gather -> alpha/beta -> (grad).  costs stay on device in w.llf.
template <typename T>
rnntStatus_t loss_op(const T* acts, T* grads, const int* labels, const int* ylen, const int* xlen, const T* gscale,
                     int V, int B, int maxT, int maxU, int blank, void* workspace, cudaStream_t s) {
    if (maxU > 1024) {
        fprintf(stderr, "rnnt_b200: maxU=%d exceeds the 1024 label positions per utterance limit\n", maxU);
        return RNNT_STATUS_INVALID_VALUE;
    }
    LossWs<T> w(workspace, B, maxT, maxU);
    const long long N = (long long)B * maxT * maxU, SK = skew_plane(maxT, maxU);
    const unsigned blocks = (unsigned)((N * 32 + 255) / 256);
    // 16-byte fast paths need float data, V % 4 == 0 and 16-byte aligned tensors (rows then stay aligned)
    const bool vec = sizeof(T) == 4 && (V % 4) == 0 && ((uintptr_t)acts % 16) == 0 && (!grads || ((uintptr_t)grads % 16) == 0);
    {
        rb::ScopedTimer tm("lse_gather_kernel", s);
        if (vec) {
            if (V <= 1024)
                rb::lse_gather_vec_kernel<8><<<blocks, 256, 0, s>>>((const float*)acts, 0, N, V, xlen, ylen, labels, maxT, maxU, SK,
                                                                    blank, (float*)w.lse, (float*)w.lpb, (float*)w.lpl);
            else
                rb::lse_gather_vec_kernel<0><<<blocks, 256, 0, s>>>((const float*)acts, 0, N, V, xlen, ylen, labels, maxT, maxU, SK,
                                                                    blank, (float*)w.lse, (float*)w.lpb, (float*)w.lpl);
        } else {
            rb::lse_gather_kernel<T><<<blocks, 256, 0, s>>>(acts, 0, N, V, xlen, ylen, labels, maxT, maxU, SK, blank,
                                                            w.lse, w.lpb, w.lpl);
        }
    }
    RB_LAUNCHED(1);
    if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    if (launch_alpha_beta(w, xlen, ylen, B, maxT, maxU, s)) return RNNT_STATUS_EXECUTION_FAILED;
    if (grads) {
        rb::ScopedTimer tm("rnnt_grad_kernel", s);
        if (vec)
            rb::rnnt_grad_vec_kernel<<<blocks, 256, 0, s>>>((const float*)acts, (float*)grads, 0, N, V, xlen, ylen, labels, maxT,
                                                            maxU, SK, blank, (const float*)w.lse, (const float*)w.alphas,
                                                            (const float*)w.betas, (const float*)w.llf, (const float*)gscale);
        else
            rb::rnnt_grad_kernel<T><<<blocks, 256, 0, s>>>(acts, grads, 0, N, V, xlen, ylen, labels, maxT, maxU, SK,
                                                           blank, w.lse, w.alphas, w.betas, w.llf, gscale);
        RB_LAUNCHED(1);
        if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    }
    return RNNT_STATUS_SUCCESS;
}

template <typename T>
rnntStatus_t compute_impl(const T* acts, T* grads, const int* labels, const int* ylen, const int* xlen, int V, int B,
                          T* costs_host, void* workspace, rnntOptions opt) {
    // argument checks of rnnt_entrypoint.cpp:49-60
    if (!acts || !labels || !ylen || !xlen || !costs_host || !workspace || V <= 0 || B <= 0 || opt.maxT <= 0 ||
        opt.maxU <= 0)
        return RNNT_STATUS_INVALID_VALUE;
    if (opt.loc == RNNT_CPU) {
        fprintf(stderr, "rnnt_b200: RNNT_CPU requested but this library has no CPU path (no fallback by design)\n");
        return RNNT_STATUS_EXECUTION_FAILED;
    }
    if (opt.loc != RNNT_GPU) return RNNT_STATUS_INVALID_VALUE;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(opt.stream);
    rnntStatus_t st = loss_op<T>(acts, grads, labels, ylen, xlen, nullptr, V, B, opt.maxT, opt.maxU, opt.blank_label,
                                 workspace, s);
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
#ifndef RNNTB200_NO_TC
            chunk_rows = 0;
            scratch_bytes = rb::tc_scratch_bytes(d);
#else
            chunk_rows = 0;
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

// C[M,N] (+)= A.B with generic strides; picks the 128x128 float4 kernel when alignment allows
template <bool AK, bool BN_>
void launch_sgemm(const float* A, const float* Bm, float* C, const float* bias, int M, int N, int K, long long sAm,
                  long long sAk, long long sBk, long long sBn, long long ldc, int accumulate, cudaStream_t s) {
    auto al16 = [](const void* p) { return ((uintptr_t)p % 16) == 0; };
    const bool a_ok = AK ? (K % 4 == 0 && sAm % 4 == 0) : (M % 4 == 0 && sAk % 4 == 0);
    const bool b_ok = BN_ ? (N % 4 == 0 && sBk % 4 == 0) : (K % 4 == 0 && sBn % 4 == 0);
    const bool fast = a_ok && b_ok && N % 4 == 0 && ldc % 4 == 0 && al16(A) && al16(Bm) && al16(C) && (!bias || al16(bias));
    if (fast) {
        // few output tiles but a long K (dW = Z^T.dL): split K over blockIdx.z so the grid fills the 132 SMs;
        // only for accumulating calls, whose output already holds valid data to atomically add into
        int splits = 1;
        const int tiles = ((N + 127) / 128) * ((M + 127) / 128);
        if (accumulate && tiles < 132 && K >= 4096) {
            splits = (132 * 4 + tiles - 1) / tiles;
            if (splits > K / 512) splits = K / 512;
            if (splits < 1) splits = 1;
        }
        dim3 grid((N + 127) / 128, (unsigned)((M + 127) / 128), splits);
        rb::sgemm128_kernel<AK, BN_><<<grid, 256, 0, s>>>(A, Bm, C, bias, M, N, K, sAm, sAk, sBk, sBn, ldc, accumulate);
    } else {
        dim3 grid((N + 63) / 64, (unsigned)((M + 63) / 64));
        rb::sgemm_kernel<AK, BN_><<<grid, 256, 0, s>>>(A, Bm, C, bias, M, N, K, sAm, sAk, sBk, sBn, ldc, accumulate);
    }
    RB_LAUNCHED(1);
}
void launch_sgemm_zw(const float* Z, const float* W, const float* bias, float* L, long long rows, int H, int V,
                     cudaStream_t s) {
    rb::ScopedTimer tm("sgemm L=Z.W+b", s);
    launch_sgemm<true, true>(Z, W, L, bias, (int)rows, V, H, H, 1, V, 1, V, 0, s);
}

rnntStatus_t exact_forward(const rnntb200JointDesc& d, const JointWs& ws, const float* enc, const float* pred,
                           const float* W, const float* bias, const int* labels, const int* ylen, const int* xlen,
                           cudaStream_t s) {
    const long long N = (long long)d.B * d.maxT * d.maxU, SK = skew_plane(d.maxT, d.maxU);
    float* Z = reinterpret_cast<float*>(ws.scratch);
    float* L = Z + ws.chunk_rows * d.H;
    for (long long r0 = 0; r0 < N; r0 += ws.chunk_rows) {
        const long long rows = (N - r0 < ws.chunk_rows) ? N - r0 : ws.chunk_rows;
        rb::zgen_kernel<<<ew_blocks(rows * d.H), 256, 0, s>>>(enc, pred, Z, r0, rows, d.maxT, d.maxU, d.H);
        RB_LAUNCHED(1);
        launch_sgemm_zw(Z, W, bias, L, rows, d.H, d.V, s);
        rb::lse_gather_kernel<float><<<(unsigned)((rows * 32 + 255) / 256), 256, 0, s>>>(
            L, r0, rows, d.V, xlen, ylen, labels, d.maxT, d.maxU, SK, d.blank_label, ws.loss.lse, ws.loss.lpb,
            ws.loss.lpl);
        RB_LAUNCHED(1);
        if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    }
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t exact_backward(const rnntb200JointDesc& d, const JointWs& ws, const float* enc, const float* pred,
                            const float* W, const float* bias, const int* labels, const int* ylen, const int* xlen,
                            const float* grad_costs, float* d_enc, float* d_pred, float* dW, float* db,
                            cudaStream_t s) {
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
        rb::zgen_kernel<<<ew_blocks(rows * d.H), 256, 0, s>>>(enc, pred, Z, r0, rows, d.maxT, d.maxU, d.H);
        launch_sgemm_zw(Z, W, bias, L, rows, d.H, d.V, s);
        // dlogits in place (gpu_rnnt_kernel.h:143-179 formula, times the upstream per-utterance gradient)
        rb::rnnt_grad_kernel<float><<<(unsigned)((rows * 32 + 255) / 256), 256, 0, s>>>(
            L, L, r0, rows, d.V, xlen, ylen, labels, d.maxT, d.maxU, SK, d.blank_label, ws.loss.lse, ws.loss.alphas,
            ws.loss.betas, ws.loss.llf, grad_costs);
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
        RB_LAUNCHED(5);
        if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    }
    return RNNT_STATUS_SUCCESS;
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
    if (!activations || !flat_labels || !label_lengths || !input_lengths || !costs_device || !workspace ||
        alphabet_size <= 0 || minibatch <= 0 || options.maxT <= 0 || options.maxU <= 0)
        return RNNT_STATUS_INVALID_VALUE;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(options.stream);
    rnntStatus_t st = loss_op<float>(activations, gradients, flat_labels, label_lengths, input_lengths, grad_scale,
                                     alphabet_size, minibatch, options.maxT, options.maxU, options.blank_label,
                                     workspace, s);
    if (st) return st;
    LossWs<float> w(workspace, minibatch, options.maxT, options.maxU);
    finish_costs_kernel<<<(minibatch + 127) / 128, 128, 0, s>>>(w.llf, w.llb, costs_device, minibatch);
    RB_LAUNCHED(1);
    return check_launch();
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
    if (!desc_ok(desc) || !enc || !pred || !W || !bias || !labels || !label_lengths || !input_lengths || !costs ||
        !workspace)
        return RNNT_STATUS_INVALID_VALUE;
    const rnntb200JointDesc& d = *desc;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(d.stream);
    JointWs ws(d, workspace);
    rnntStatus_t st;
    if (d.precision == RNNTB200_FP32_EXACT) {
        st = exact_forward(d, ws, enc, pred, W, bias, labels, label_lengths, input_lengths, s);
    } else {
#ifndef RNNTB200_NO_TC
        unsigned nl = 0;
        st = rb::tc_forward(d, ws.scratch, enc, pred, W, bias, labels, label_lengths, input_lengths, ws.loss.lse,
                            ws.loss.lpb, ws.loss.lpl, s, &nl);
        RB_LAUNCHED(nl);
#else
        fprintf(stderr, "rnnt_b200: built without the tensor-core path\n");
        st = RNNT_STATUS_EXECUTION_FAILED;
#endif
    }
    if (st) return st;
    st = launch_alpha_beta(ws.loss, input_lengths, label_lengths, d.B, d.maxT, d.maxU, s);
    if (st) return st;
    const int* overflow = nullptr;
#ifndef RNNTB200_NO_TC
    if (d.precision != RNNTB200_FP32_EXACT) {      // the keeping forward ranked the tiles: its overflow word is fresh
        const rb::TcScratch sc = rb::tc_scratch_layout(d, ws.scratch);
        if (rb::tc_keep(d, sc)) overflow = sc.count + 1;
    }
#endif
    finish_costs_kernel<<<(d.B + 127) / 128, 128, 0, s>>>(ws.loss.llf, ws.loss.llb, costs, d.B, overflow);
    RB_LAUNCHED(1);
    return check_launch();
}

rnntStatus_t rnntb200_joint_loss_backward(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                          const float* W, const float* bias, const int* labels,
                                          const int* label_lengths, const int* input_lengths,
                                          const float* grad_costs, float* d_enc, float* d_pred, float* dW,
                                          float* db, void* workspace) {
    if (!desc_ok(desc) || !enc || !pred || !W || !bias || !labels || !label_lengths || !input_lengths ||
        !grad_costs || !d_enc || !d_pred || !dW || !db || !workspace)
        return RNNT_STATUS_INVALID_VALUE;
    const rnntb200JointDesc& d = *desc;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(d.stream);
    JointWs ws(d, workspace);
    if (d.precision == RNNTB200_FP32_EXACT)
        return exact_backward(d, ws, enc, pred, W, bias, labels, label_lengths, input_lengths, grad_costs, d_enc,
                              d_pred, dW, db, s);
#ifndef RNNTB200_NO_TC
    unsigned nl = 0;
    const rb::LossPlanes lp{ws.loss.lse, ws.loss.lpb, ws.loss.lpl, ws.loss.alphas, ws.loss.betas, ws.loss.llf};
    rnntStatus_t st = rb::tc_backward(d, ws.scratch, enc, pred, bias, labels, label_lengths, input_lengths, lp, grad_costs,
                                      d_enc, d_pred, dW, db, s, &nl);
    RB_LAUNCHED(nl);
    return st;
#else
    fprintf(stderr, "rnnt_b200: built without the tensor-core path\n");
    return RNNT_STATUS_EXECUTION_FAILED;
#endif
}

rnntStatus_t rnntb200_joint_logits(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                   const float* W, const float* bias, float* logits, void* workspace) {
    if (!desc_ok(desc) || !enc || !pred || !W || !bias || !logits || !workspace) return RNNT_STATUS_INVALID_VALUE;
    rnntb200JointDesc d = *desc;
    d.precision = RNNTB200_FP32_EXACT;  // the materialising entry is the fp32 literal of model.py:158-166
    cudaStream_t s = reinterpret_cast<cudaStream_t>(d.stream);
    JointWs ws(d, workspace);
    const long long N = (long long)d.B * d.maxT * d.maxU;
    float* Z = reinterpret_cast<float*>(ws.scratch);
    for (long long r0 = 0; r0 < N; r0 += ws.chunk_rows) {
        const long long rows = (N - r0 < ws.chunk_rows) ? N - r0 : ws.chunk_rows;
        rb::zgen_kernel<<<ew_blocks(rows * d.H), 256, 0, s>>>(enc, pred, Z, r0, rows, d.maxT, d.maxU, d.H);
        launch_sgemm_zw(Z, W, bias, logits + r0 * d.V, rows, d.H, d.V, s);
        RB_LAUNCHED(1);
        if (check_launch()) return RNNT_STATUS_EXECUTION_FAILED;
    }
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t rnntb200_joint_step(const float* f, long long ldf, const float* g, long long ldg, const float* K1,
                                 const float* b1, const float* K2, const float* b2, int B, int P, int H, int V,
                                 float* logits, int* best, float* best_logp, CUstream stream) {
    if (!f || !g || !K2 || B <= 0 || P <= 0 || H <= 0 || V <= 0 || (!logits && !best && !best_logp)) return RNNT_STATUS_INVALID_VALUE;
    if (!K1 && P != H) return RNNT_STATUS_INVALID_VALUE;
    if (P > rb::STEP_MAX_DIM || H > rb::STEP_CLUSTER * rb::STEP_THREADS || V > (1 << 20)) {
        fprintf(stderr, "rnnt_b200: rnntb200_joint_step supports P <= %d, H <= %d\n", rb::STEP_MAX_DIM, rb::STEP_CLUSTER * rb::STEP_THREADS);
        return RNNT_STATUS_INVALID_VALUE;
    }
    rb::StepParams p{f, g, ldf, ldg, K1, b1, K2, b2, B, P, H, V, logits, best, best_logp};
    const size_t smem = rb::joint_step_smem(P, H, V);
    if (smem > 48 * 1024 && !rb::tc_smem_optin(reinterpret_cast<const void*>(rb::joint_step_kernel))) return RNNT_STATUS_EXECUTION_FAILED;
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
        rb::colsum_add_kernel<<<(H + 31) / 32, 256, 0, s>>>(dA, rows, H, db1);
        RB_LAUNCHED(1);
    }
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
