/** \file rnnt_b200.h
 *  C ABI of librnnt_b200.so -- the H100-native (sm_90a) RNN-T loss hot path.
 *
 *  Part 1 is a drop-in for the warp-transducer C interface the reference application binds
 *  (reference: warp-transducer/include/rnnt.h:16-143, implemented in
 *  warp-transducer/src/rnnt_entrypoint.cpp:14-185): same symbol names, argument order, status
 *  codes and by-value options struct, so the reference's TensorFlow op
 *  (tensorflow_binding/src/warprnnt_op.cc:105-141) or PyTorch binding
 *  (pytorch_binding/src/binding.cpp:84-154) links against this library unchanged.
 *
 *  Part 2 adds the entry points the reference has no analogue for: the fused joint-network +
 *  loss path (model.py:158-166 -> utils/loss.py:24-36 -> warp-transducer) in which the
 *  (B,T,U,V) fp32 logits are never written to HBM.  They follow the same conventions: status enum,
 *  caller-owned device workspace sized by a pure function, explicit CUstream.  The Part 2 calls are
 *  stream-ordered: no device allocation, no host synchronisation and no read-back (the only host
 *  synchronisation in the library is the one the reference's contract mandates at the end of
 *  compute_rnnt_loss: costs are host memory, gpu_rnnt.h:209-213).  State kept by the library:
 *  a per-(device, kernel) flag that the >48 KB dynamic shared memory opt-in has been set
 *  (mutex-protected; any number of devices and host threads per process), the launch counter and the
 *  optional timing records of rnntb200_set_timing.
 *
 *  What reaches HBM on the tensor-core path (N = lattice cells, V vocabulary):
 *    keep_activations = 0  forward: lse + two log-probs per cell, alpha, beta (O(N) floats).  The backward
 *                          re-runs the projection per utterance chunk, leaving 2 bytes per logit (bf16 softmax
 *                          numerators relative to one fp32 reference per lattice row) in the workspace for the two
 *                          gradient GEMM kernels to consume; no (B,T,U,V) tensor is produced by the forward call.
 *    keep_activations = 1  the forward itself writes those numerators (one pass fewer on the tensor cores).
 *    In both modes the logit gradients, dZ and z = tanh(enc+pred) exist only in shared / tensor memory.
 *
 *  There is NO CPU implementation in this library: loc == RNNT_CPU returns
 *  RNNT_STATUS_EXECUTION_FAILED (and says so on stderr) instead of silently falling back.
 */
#pragma once

#ifdef __cplusplus
#include <cstddef>
extern "C" {
#else
#include <stddef.h>
#include <stdbool.h>
#endif

/* forward declaration of the CUDA typedef (rnnt.h:13) */
typedef struct CUstream_st* CUstream;

/* ------------------------------------------------------------------------------------------
 * Part 1 -- warp-transducer compatible surface
 * ------------------------------------------------------------------------------------------ */

/** rnnt.h:16-22 */
typedef enum {
    RNNT_STATUS_SUCCESS = 0,
    RNNT_STATUS_MEMOPS_FAILED = 1,
    RNNT_STATUS_INVALID_VALUE = 2,
    RNNT_STATUS_EXECUTION_FAILED = 3,
    RNNT_STATUS_UNKNOWN_ERROR = 4
} rnntStatus_t;

/** rnnt.h:33-36 */
typedef enum { RNNT_CPU = 0, RNNT_GPU = 1 } rnntComputeLocation;

/** rnnt.h:43-64 -- 32 bytes on x86-64, passed BY VALUE.  batch_first is ignored by the GPU
 *  path exactly as in the reference (rnnt_entrypoint.cpp:75-76 never forwards it). */
struct rnntOptions {
    rnntComputeLocation loc;
    unsigned int num_threads;
    CUstream stream;
    int blank_label;
    int maxT;
    int maxU;
    bool batch_first;
};
#ifndef __cplusplus
typedef struct rnntOptions rnntOptions;
#endif

/** rnnt.h:25 / rnnt_entrypoint.cpp:14-16 -- API version, returns 1. */
int get_warprnnt_version();

/** rnnt.h:31 / rnnt_entrypoint.cpp:18-35 -- same five strings. */
const char* rnntGetStatusString(rnntStatus_t status);

/** rnnt.h:138-142 / rnnt_entrypoint.cpp:96-128.
 *  gpu == false returns the reference's CPU figure B*4*maxT*maxU*dtype (kept for host-logic
 *  parity; this library never uses a CPU workspace).  gpu == true returns what THIS library
 *  needs for compute_rnnt_loss: B*(4*SK + maxT*maxU + 2)*dtype with SK = (maxT+maxU-1)*maxU
 *  (diagonal-major lp_blank / lp_label / alpha / beta planes, the lse plane and the two
 *  log-likelihood vectors) -- larger than the reference's B*(3*maxT*maxU+2)*dtype, which is
 *  why callers must size the workspace through this function, as the reference's bindings do
 *  (warprnnt_op.cc:105-128, binding.cpp:120-137). */
rnntStatus_t get_workspace_size(int maxT, int maxU, int minibatch, bool gpu, size_t* size_bytes,
                                size_t dtype_size
#ifdef __cplusplus
                                = sizeof(float)
#endif
);

/** rnnt.h:104-113 / rnnt_entrypoint.cpp:38-93, GPU semantics (gpu_rnnt.h:82-215):
 *  activations  device, raw logits (B,maxT,maxU,V) row-major, softmax done inside
 *  gradients    device, same shape, or NULL for forward-only; padded cells are written 0
 *  flat_labels  DEVICE int32 (B, maxU-1) row-major (warprnnt_op.cc:88-94,193-195)
 *  label_lengths, input_lengths  DEVICE int32 (B)
 *  costs        HOST float (B): copied back and negated after a stream synchronise, as
 *               gpu_rnnt.h:209-213 does.  (rnntb200_loss_device below keeps them on device.)
 *  workspace    device, get_workspace_size(..., gpu=true) bytes
 *  Limits: maxU <= 1024 (one thread per label position, same bound as gpu_rnnt.h:127).
 *  Errors: NULL / non-positive arguments -> RNNT_STATUS_INVALID_VALUE (rnnt_entrypoint.cpp:49-60);
 *  CUDA launch failure -> RNNT_STATUS_EXECUTION_FAILED; copy failure -> RNNT_STATUS_MEMOPS_FAILED;
 *  loc == RNNT_CPU -> RNNT_STATUS_EXECUTION_FAILED (no CPU fallback). */
rnntStatus_t compute_rnnt_loss(const float* const activations, float* gradients, const int* const flat_labels,
                               const int* const label_lengths, const int* const input_lengths, int alphabet_size,
                               int minibatch, float* costs, void* workspace, rnntOptions options);

/** rnnt.h:115-124 / rnnt_entrypoint.cpp:130-185 -- double-precision twin. */
rnntStatus_t compute_rnnt_loss_fp64(const double* const activations, double* gradients,
                                    const int* const flat_labels, const int* const label_lengths,
                                    const int* const input_lengths, int alphabet_size, int minibatch,
                                    double* costs, void* workspace, rnntOptions options);

/* ------------------------------------------------------------------------------------------
 * Part 2 -- B200 additions (no reference analogue; conventions as above)
 * ------------------------------------------------------------------------------------------ */

/** compute_rnnt_loss with DEVICE costs and no host synchronisation.  This is
 *  what the torch surface calls; replaces the D2H + cudaStreamSynchronize of gpu_rnnt.h:209-213.
 *  grad_scale: optional DEVICE float (B); when non-NULL gradients[b] are pre-multiplied by it
 *  (folds _RNNTLossGrad's grad_loss[:,None,None,None]*grads, warprnnt_tensorflow/__init__.py:37-42). */
rnntStatus_t rnntb200_loss_device(const float* activations, float* gradients, const int* flat_labels,
                                  const int* label_lengths, const int* input_lengths, const float* grad_scale,
                                  int alphabet_size, int minibatch, float* costs_device, void* workspace,
                                  rnntOptions options);

/** FastEmit regularisation (Yu et al., "FastEmit: Low-latency Streaming ASR with Sequence-level Emission
 *  Regularization", ICASSP 2021) on the entries that form gradients.  fastemit_lambda >= 0, finite, one value for the
 *  batch: the gradient of every label-emission log-probability lp_label(t,u) is multiplied by (1 + lambda), blank
 *  log-probabilities keep theirs.  w.r.t. the logits (softmax inside), with occupancy gamma, blank-arc term gamma_B and
 *  label-arc occupancy gamma_L of a cell:
 *    d cost / d logit[v] = (gamma + lambda*gamma_L) p_v - [v == blank] gamma_B - [v == label_u] (1 + lambda) gamma_L.
 *  The COSTS ARE UNCHANGED (-log p(y|x), not (1 + lambda) times it), so loss curves compare across lambda.
 *  fastemit_lambda == 0 gives results bit-identical to the entries without the suffix, which are these entries with 0.
 *  A negative, NaN or infinite fastemit_lambda returns RNNT_STATUS_INVALID_VALUE before any device work. */
rnntStatus_t rnntb200_loss_device_fastemit(const float* activations, float* gradients, const int* flat_labels,
                                           const int* label_lengths, const int* input_lengths, const float* grad_scale,
                                           int alphabet_size, int minibatch, float* costs_device, void* workspace,
                                           rnntOptions options, float fastemit_lambda);

/** Element type of 16-bit logits (mixed-precision training: fp16 / bf16 activations). */
typedef enum {
    RNNTB200_LOGITS_F16 = 0,  /**< IEEE binary16 */
    RNNTB200_LOGITS_BF16 = 1  /**< bfloat16 */
} rnntb200LogitType;

/** rnntb200_loss_device on 16-bit logits, split into a forward and a backward call so that the gradient is formed
 *  only when it is asked for, with the upstream gradient multiplied in before its one rounding to 16 bits (an fp16
 *  gradient of an unscaled cost underflows; a loss-scaled one does not).
 *  activations  device, raw logits (B,maxT,maxU,V) row-major of type logit_type, softmax done inside
 *  costs_device device float (B): -log p(y|x) per utterance
 *  workspace    device, get_workspace_size(maxT, maxU, B, true, &sz, 4) bytes: the fp32 planes of the loss op.  The
 *               forward fills it; the backward reads it and must get it unchanged.
 *  All arithmetic is fp32: each logit is converted exactly on load, each gradient rounded to nearest-even on store.
 *  Stream-ordered, no allocation, no host synchronisation (CUDA-graph capturable).  Errors: NULL pointers,
 *  non-positive sizes, maxU > 1024, a blank outside [0, V) or an unknown logit_type -> RNNT_STATUS_INVALID_VALUE. */
rnntStatus_t rnntb200_loss16_forward(const void* activations, int logit_type, const int* flat_labels,
                                     const int* label_lengths, const int* input_lengths, int alphabet_size, int minibatch,
                                     float* costs_device, void* workspace, rnntOptions options);

/** Backward of rnntb200_loss16_forward (same activations, labels, lengths, options and workspace):
 *  gradients (B,maxT,maxU,V) of type logit_type, device, OVERWRITTEN = grad_costs[b] * d(costs[b])/d(activations) in
 *  one pass; padded cells are written 0.  grad_costs: optional DEVICE float (B), NULL means 1 (as grad_scale of
 *  rnntb200_loss_device). */
rnntStatus_t rnntb200_loss16_backward(const void* activations, int logit_type, const int* flat_labels,
                                      const int* label_lengths, const int* input_lengths, const float* grad_costs,
                                      int alphabet_size, int minibatch, void* gradients, const void* workspace,
                                      rnntOptions options);

/** rnntb200_loss16_backward with FastEmit (see rnntb200_loss_device_fastemit); the forward call is unchanged. */
rnntStatus_t rnntb200_loss16_backward_fastemit(const void* activations, int logit_type, const int* flat_labels,
                                               const int* label_lengths, const int* input_lengths, const float* grad_costs,
                                               int alphabet_size, int minibatch, void* gradients, const void* workspace,
                                               rnntOptions options, float fastemit_lambda);

typedef enum {
    RNNTB200_FP32_EXACT = 0, /**< fp32 CUDA-core arithmetic; parity gate rtol 1e-4 (BASELINE C1/C2) */
    RNNTB200_BF16_TC = 1     /**< 16-bit operands on wgmma tensor cores, fp32 accumulate (BASELINE C3-C5): the forward
                                  projection runs on fp16 z / W (11-bit significands), the two gradient GEMMs on bf16 */
} rnntb200Precision;

/** Problem descriptor of the fused joint + loss path (model.py:158-166 hoisted form, SURVEY 8a2):
 *    z[b,t,u,:]  = tanh(enc[b,t,:] + pred[b,u,:])            model.py:158-163
 *    logits      = z . W + bias,  W is (H,V) row-major        model.py:165-166
 *    costs[b]    = RNN-T NLL of logits[b] (softmax inside)    utils/loss.py:24-36
 *  RNNTB200_BF16_TC requires H % 64 == 0, 64 <= H <= 768 and V % 64 == 0. */
typedef struct {
    int B, maxT, maxU, H, V;
    int blank_label;
    int precision; /* rnntb200Precision */
    CUstream stream;
    /** 0: unknown.  N > 0: the caller promises that at most N of the batch's 16 x 8 lattice tiles intersect the valid lattice,
     *  N >= sum_b ceil(T_b / 16) * ceil((U_b + 1) / 8) with U_b = label_lengths[b] (a host-side sum over lengths the data
     *  loader has anyway); with the windows of the _windowed entries, at most N tiles are valid under their rule.  The kept numerators are indexed by compact tile slots, but only the device knows how many tiles
     *  are valid (the library never synchronises with the host), so by default the workspace is sized for every tile of
     *  the padded (maxT, maxU) lattice and a batch whose padded numerators exceed 16 GiB is processed in utterance chunks,
     *  which rules keep_activations out.  With a bound the workspace holds N row blocks and the batch is one chunk.  If
     *  the promise is broken nothing is written out of bounds: the forward prints an error and returns NaN costs.
     *  (Round 1 had `allow_host_sync` here: same offset and type, 0 keeps the old behaviour.) */
    int valid_tile_bound;
    /** 0: nothing but lse / log-prob pairs / alpha / beta survives the forward; the backward re-runs the projection
     *  chunk by chunk.  1 (tensor-core path): the forward also leaves, in the workspace, the softmax numerators of
     *  every lattice cell as bf16 (2 bytes per logit) and one fp32 reference per lattice row; the backward then skips its own
     *  projection pass.  Set it when a backward call will follow; it is honoured only when the whole batch fits one
     *  workspace chunk (<= 16 GiB of numerators), otherwise (and for fp32) ignored.  Must have the same value in the
     *  forward and the backward call. */
    int keep_activations;
} rnntb200JointDesc;

/** Bytes of device workspace the forward/backward pair needs (pure function of the descriptor).  On the tensor-core
 *  path this includes, besides the kept numerators the chunk plan is sized by, the dW GEMM's bf16 operand: (H + 64) * 2
 *  bytes per kept lattice row, not counted against the 16 GiB chunk budget or the 56 GiB valid_tile_bound rule
 *  (2.95 GB at B=32 T=512 U=128 H=640, on top of 4.7 GB of numerators). */
rnntStatus_t rnntb200_joint_workspace_size(const rnntb200JointDesc* desc, size_t* size_bytes);

/** Forward: enc (B,maxT,H), pred (B,maxU,H), W (H,V), bias (V) fp32 device; labels (B,maxU-1),
 *  label_lengths (B), input_lengths (B) int32 device; costs (B) fp32 DEVICE.  Leaves lse, the
 *  cached log-prob pairs, alpha and beta in `workspace` for the backward call. */
rnntStatus_t rnntb200_joint_loss_forward(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                         const float* W, const float* bias, const int* labels,
                                         const int* label_lengths, const int* input_lengths, float* costs,
                                         void* workspace);

/** Backward through the loss and the joint (run_rnnt.py:284's tape.gradient for this path):
 *  grad_costs (B) device = d(total)/d(costs[b]) (1/B for run_rnnt.py:278);
 *  outputs d_enc (B,maxT,H), d_pred (B,maxU,H), dW (H,V), db (V): fp32 device, OVERWRITTEN.
 *  Must follow a forward call with the same descriptor, inputs and workspace. */
rnntStatus_t rnntb200_joint_loss_backward(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                          const float* W, const float* bias, const int* labels,
                                          const int* label_lengths, const int* input_lengths,
                                          const float* grad_costs, float* d_enc, float* d_pred, float* dW,
                                          float* db, void* workspace);

/** rnntb200_joint_loss_backward with FastEmit (see rnntb200_loss_device_fastemit), on both precisions; the forward call
 *  is unchanged and the descriptor keeps its layout. */
rnntStatus_t rnntb200_joint_loss_backward_fastemit(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                                   const float* W, const float* bias, const int* labels,
                                                   const int* label_lengths, const int* input_lengths,
                                                   const float* grad_costs, float* d_enc, float* d_pred, float* dW,
                                                   float* db, void* workspace, float fastemit_lambda);

/** Alignment-restricted RNN-T (Mahadeokar et al., "Alignment Restricted Streaming Recurrent Neural Network Transducer",
 *  SLT 2021): the loss sums only over the paths that stay inside per-label time windows.  Per utterance b and lattice
 *  column u in [0, U_b), U_b = label_lengths[b] + 1, the caller gives an inclusive frame window [t_lo[b,u], t_hi[b,u]]:
 *  two int32 DEVICE arrays (B, maxU), row stride maxU, entries at u >= U_b ignored.  Cell (t,u) is ALLOWED iff
 *  t_lo[b,u] <= t <= t_hi[b,u] and t < T_b.  Any int32 is accepted and nothing is clamped: t_lo > t_hi, or a window outside
 *  [0, T_b), is an empty column.  BOTH ARCS LEAVING A CELL THAT IS NOT ALLOWED HAVE LOG-PROBABILITY -inf, as does the
 *  terminating blank at (T_b-1, U_b-1) if that cell is not allowed; equivalently
 *    costs[b] = -log sum P(path) over the paths that visit allowed cells only.
 *  Everything else (softmax inside, blank, labels, grad_costs, FastEmit's (1 + lambda) on label arcs, padded cells written
 *  0) is as in the entries without windows.  Consequences:
 *    - the gradients of the logits of a cell that is not allowed are exactly 0;
 *    - windows that cover the lattice (t_lo <= 0, t_hi >= T_b - 1) give costs and gradients bit-identical to the entries
 *      without windows, which are these entries with t_lo == t_hi == NULL;
 *    - windows that admit no path give costs[b] = +inf and exactly-zero gradients for that utterance, no NaN, and leave
 *      the other utterances of the batch untouched.
 *  The forward AND the backward entry take the windows (they change the costs), and must be given the same ones.
 *  Exactly one of t_lo / t_hi NULL -> RNNT_STATUS_INVALID_VALUE before any device work.
 *  On the tensor-core joint path a 16 x 8 lattice tile (b, t0, u0) is VALID iff it intersects the T_b x U_b lattice and
 *  some column u in [u0, min(u0 + 8, U_b)) has [t_lo, t_hi] meet [t0, t0 + 16); tiles that are not valid are never
 *  computed, in the forward or in either backward GEMM, and take no room among the kept numerators.
 *  rnntb200JointDesc.valid_tile_bound keeps its meaning under this rule ("at most N tiles are valid"; a broken promise
 *  gives NaN costs and no out-of-bounds write).  The loss op and the fp32 joint path skip the logits of cells that are not
 *  allowed in their softmax and gradient passes (the fp32 joint path still projects them).
 *  rnntb200_loss_device_windowed: rnntb200_loss_device_fastemit with windows. */
rnntStatus_t rnntb200_loss_device_windowed(const float* activations, float* gradients, const int* flat_labels,
                                           const int* label_lengths, const int* input_lengths, const float* grad_scale,
                                           const int* t_lo, const int* t_hi, int alphabet_size, int minibatch,
                                           float* costs_device, void* workspace, rnntOptions options,
                                           float fastemit_lambda);

/** rnntb200_loss16_forward / rnntb200_loss16_backward_fastemit with windows (see rnntb200_loss_device_windowed). */
rnntStatus_t rnntb200_loss16_forward_windowed(const void* activations, int logit_type, const int* flat_labels,
                                              const int* label_lengths, const int* input_lengths, const int* t_lo,
                                              const int* t_hi, int alphabet_size, int minibatch, float* costs_device,
                                              void* workspace, rnntOptions options);
rnntStatus_t rnntb200_loss16_backward_windowed(const void* activations, int logit_type, const int* flat_labels,
                                               const int* label_lengths, const int* input_lengths, const int* t_lo,
                                               const int* t_hi, const float* grad_costs, int alphabet_size, int minibatch,
                                               void* gradients, const void* workspace, rnntOptions options,
                                               float fastemit_lambda);

/** rnntb200_joint_loss_forward / rnntb200_joint_loss_backward_fastemit with windows (see rnntb200_loss_device_windowed),
 *  both precisions; the descriptor keeps its layout.  The windowed backward is as deterministic as the plain one. */
rnntStatus_t rnntb200_joint_loss_forward_windowed(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                                  const float* W, const float* bias, const int* labels,
                                                  const int* label_lengths, const int* input_lengths, const int* t_lo,
                                                  const int* t_hi, float* costs, void* workspace);
rnntStatus_t rnntb200_joint_loss_backward_windowed(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                                   const float* W, const float* bias, const int* labels,
                                                   const int* label_lengths, const int* input_lengths, const int* t_lo,
                                                   const int* t_hi, const float* grad_costs, float* d_enc, float* d_pred,
                                                   float* dW, float* db, void* workspace, float fastemit_lambda);

/** Forced alignment: the single most likely path through the lattice the loss sums over (Viterbi), per utterance b
 *  with T = input_lengths[b], U = label_lengths[b] + 1 and the log-probs of the loss, lpb(t,u) at blank and lpl(t,u)
 *  at labels[b][u]:
 *    delta(0,0) = 0
 *    delta(t,u) = max(delta(t-1,u) + lpb(t-1,u), delta(t,u-1) + lpl(t,u-1))   (a predecessor outside the lattice: -inf)
 *    best_logp[b] = delta(T-1,U-1) + lpb(T-1,U-1)  <=  -costs[b]
 *  Ties: the label arc wins only when it is STRICTLY greater, so on an exact tie the blank predecessor wins -- among
 *  equally scoring paths the one that emits every label earliest.
 *  label_frames (B, maxU-1) int32 device, row stride maxU-1: label_frames[b][j] is the frame t at which the best path
 *  takes the label arc (t,j) -> (t,j+1), i.e. emits labels[b][j]; -1 for j >= U-1.  Per utterance the frames are
 *  non-decreasing and lie in [0, T).  label_frames may be NULL only when maxU == 1.
 *  costs / best_logp (B) float device.  The costs are those of the matching forward entry, bit for bit.
 *  Not differentiable; the workspace (same size as the forward's) is overwritten with the decisions and cannot feed a
 *  backward call.  Stream-ordered, no allocation, no host synchronisation (CUDA-graph capturable).  Errors as the
 *  matching forward entry, plus maxU > 1024 and a blank outside [0, V) -> RNNT_STATUS_INVALID_VALUE before any device
 *  work.
 *  rnntb200_align_device: fp32 logits, arguments of rnntb200_loss_device (workspace of get_workspace_size). */
rnntStatus_t rnntb200_align_device(const float* activations, const int* flat_labels, const int* label_lengths,
                                   const int* input_lengths, int alphabet_size, int minibatch, float* costs_device,
                                   float* best_logp, int* label_frames, void* workspace, rnntOptions options);

/** Forced alignment on 16-bit logits (arguments of rnntb200_loss16_forward; fp32 arithmetic). */
rnntStatus_t rnntb200_align16(const void* activations, int logit_type, const int* flat_labels, const int* label_lengths,
                              const int* input_lengths, int alphabet_size, int minibatch, float* costs_device,
                              float* best_logp, int* label_frames, void* workspace, rnntOptions options);

/** Forced alignment on the fused joint path (arguments of rnntb200_joint_loss_forward, workspace of
 *  rnntb200_joint_workspace_size), both precisions; the (B,T,U,V) logits are never written.  keep_activations is
 *  ignored (nothing is kept).  valid_tile_bound is honoured: a broken promise gives NaN costs, NaN best_logp and
 *  label_frames of -1. */
rnntStatus_t rnntb200_joint_align(const rnntb200JointDesc* desc, const float* enc, const float* pred, const float* W,
                                  const float* bias, const int* labels, const int* label_lengths,
                                  const int* input_lengths, float* costs, float* best_logp, int* label_frames,
                                  void* workspace);

/** Joint network forward only, materialising logits (B,maxT,maxU,V) fp32 -- the literal
 *  model.py:158-166 output, used by the drop-in `Joint` module when a caller wants the tensor
 *  (e.g. to feed rnnt_loss/compute_rnnt_loss exactly as run_rnnt.py:269-273 does). */
rnntStatus_t rnntb200_joint_logits(const rnntb200JointDesc* desc, const float* enc, const float* pred,
                                   const float* W, const float* bias, float* logits, void* workspace);

/** Greedy-decode joint (utils/decoding.py:6-18, called per step at :69-78): one lattice cell per batch row,
 *    logits[b,:] = tanh((f[b,:] + g[b,:]) . K1 + b1) . K2 + b2;  best[b] = argmax_v logits (smallest index among equal
 *    maxima, as tf.argmax);  best_logp[b] = log_softmax(logits[b])[best[b]]
 *  in ONE launch (thread-block clusters of 8 CTAs per row; fp32 FMA arithmetic).  f, g: (B,P) device rows with strides
 *  ldf, ldg (so f = encoded[:, i, :] and g = pred_out[:, -1, :] need no copy); K1 (P,H) and b1 (H) are Keras Dense-1
 *  (K1 == NULL: f, g are the already projected activations, P == H); K2 (H,V), b2 (V).  Any of logits (B,V), best (B),
 *  best_logp (B) may be NULL, not all.
 *  Non-finite logits: a NaN outranks every number and the first NaN wins (as np.argmax / torch.argmax), so best[b] always
 *  lies in [0, V) -- 0 for a row of -inf.  best_logp[b] is NaN for a row that holds a NaN or only -inf.
 *  Limits: P <= 4096, H <= 2048 and V <= 8 * (58088 - max(P, 256) - H - 256): each CTA holds its eighth of the logits in
 *  shared memory, 4 * (max(P, 256) + H + 256 + ceil(V / 8)) bytes within the 227 KB per block of sm_90 (V <= 460096 at
 *  P = H = 64, 413504 at P = 4096, H = 2048).  Past them: RNNT_STATUS_INVALID_VALUE before any device work. */
rnntStatus_t rnntb200_joint_step(const float* f, long long ldf, const float* g, long long ldg, const float* K1,
                                 const float* b1, const float* K2, const float* b2, int B, int P, int H, int V,
                                 float* logits, int* best, float* best_logp, CUstream stream);

/** Dense-1 of the joint (model.py:162-163, Keras kernel (P,H) + bias (H)) applied BEFORE the broadcast add -- it is linear in
 *  front of its tanh, so W1^T (f_t + g_u) + b1 = (W1^T f_t + b1) + W1^T g_u (SURVEY 8 a2): the hot path's inputs
 *  enc_acts / pred_acts are these two projections.
 *    forward:   out[r,:] = X[r,:] . K1 (+ b1)                       X (rows,P) -> out (rows,H), b1 may be NULL (the pred side)
 *    backward:  dX = dA . K1^T;  dK1 += X^T . dA;  db1 += sum_r dA[r,:]      (dX, dK1, db1 may each be NULL; dK1 / db1 are
 *               ACCUMULATED into, so the encoder-side and the prediction-side call add into one zeroed buffer)
 *  fp32 FMA kernels of this library (no GEMM library).  dK1 is a split-K product combined with float atomics: its last bits
 *  depend on the order the partial sums arrive in (as the exact fp32 path's dW).  1 <= rows <= INT_MAX (X may exceed 2^31
 *  elements; a product taller than one launch's 65535 row tiles runs as several launches), else
 *  RNNT_STATUS_INVALID_VALUE, as for dX without K1 and dK1 without X. */
rnntStatus_t rnntb200_dense1_forward(const float* X, long long rows, int P, const float* K1, const float* b1, int H,
                                     float* out, CUstream stream);
rnntStatus_t rnntb200_dense1_backward(const float* X, const float* dA, const float* K1, long long rows, int P, int H,
                                      float* dX, float* dK1, float* db1, CUstream stream);

/* ------------------------------------------------------------------------------------------
 * Part 3 -- pruned RNN-T (Kuang, Guo, Kang, Lin, Povey, "Pruned RNN-T for fast, memory-efficient ASR training",
 * Interspeech 2022): the trivial joiner's "simple" loss and the band it chooses for the full joint
 * ------------------------------------------------------------------------------------------ */

/** The simple loss: am (B,maxT,V) and lm (B,maxU,V) fp32 device, row-major; labels (B,maxU-1), label_lengths (B),
 *  input_lengths (B) int32 device; options.blank_label / maxT / maxU / stream as in rnntb200_loss16_forward (loc and
 *  num_threads are ignored).  The cost is the ordinary RNN-T loss, softmax inside, over the logits
 *    x[b,t,u,:] = am[b,t,:] + lm[b,u,:]
 *  i.e. rnntb200_loss_device on am[:,:,None,:] + lm[:,None,:,:], without that (B,T,U,V) tensor ever being formed: the
 *  log-softmax normaliser factorises into exp(am - max) . exp(lm - max)^T, an fp32 FMA GEMM per utterance.  A cell whose
 *  factorised normaliser falls below 2^-64 (am's and lm's large entries in different columns) takes a direct log-sum-exp
 *  over V instead, and its exact softmax in the backward: costs stay finite however far apart the two peaks are.
 *  Workspace: rnntb200_simple_workspace_size bytes (a pure function).  No FastEmit and no windows on this loss.
 *  Stream-ordered, no allocation, no host synchronisation, CUDA-graph capturable; no float atomics (bit-identical reruns).
 *  Errors: NULL pointers, non-positive sizes, maxU > 1024 or a blank outside [0, V) -> RNNT_STATUS_INVALID_VALUE before
 *  any device work. */
rnntStatus_t rnntb200_simple_workspace_size(int B, int maxT, int maxU, int V, size_t* size_bytes);

/** Forward: costs (B) fp32 DEVICE, -log p(y|x) of the simple lattice; leaves its planes in the workspace. */
rnntStatus_t rnntb200_simple_loss_forward(const float* am, const float* lm, const int* labels, const int* label_lengths,
                                          const int* input_lengths, int V, int B, float* costs, void* workspace,
                                          rnntOptions options);

/** Backward on the forward's unchanged workspace (which it leaves unchanged for the windows call):
 *  d_am[b,t,:] = sum_u grad_costs[b] dx[b,t,u,:] and d_lm[b,u,:] = sum_t grad_costs[b] dx[b,t,u,:], fp32 device,
 *  OVERWRITTEN; rows at t >= T_b or u >= U_b are exactly 0.  grad_costs: optional DEVICE float (B), NULL means 1. */
rnntStatus_t rnntb200_simple_loss_backward(const float* am, const float* lm, const int* labels, const int* label_lengths,
                                           const int* input_lengths, int V, int B, const float* grad_costs, float* d_am,
                                           float* d_lm, void* workspace, rnntOptions options);

/** The pruning band of the forward's simple lattice (DESIGN §1), as the per-column frame windows of the _windowed entries:
 *  with S = s_range >= 2 and gamma_B / gamma_L the blank- and label-arc occupancies,
 *    score(t,s) = sum_{u=s}^{min(s+S,U_b)-1} gamma_B(t,u) - gamma_L(t,s-1),  s in [0, max(0, U_b - S)];
 *  s_t its smallest argmax for t < T_b - 1 and s_{T_b-1} = max(0, U_b - S); then s_t <- min_{t' >= t} s_t' and
 *  s_t <- min((S-1) t, max_{t' >= t} (s_t' - (S-1)(t' - t))).  Cell (t,u) is in the band iff s_t <= u < s_t + S, and
 *    t_lo[b,u] = min{t < T_b : s_t <= u < s_t + S},  t_hi[b,u] = max{...}   (int32 DEVICE (B, maxU)),
 *  (0, -1) for u >= U_b and for a column no frame's band reaches.  The band admits a path iff (S-1) T_b >= U_b - 1;
 *  S >= U_b gives full windows.  Reads the forward's planes and does not modify them; uses the workspace's own band
 *  planes.  Errors: NULL pointers, B <= 0, s_range < 2, maxU > 1024 -> RNNT_STATUS_INVALID_VALUE. */
rnntStatus_t rnntb200_simple_prune_windows(const int* label_lengths, const int* input_lengths, int B, int s_range,
                                           int* t_lo, int* t_hi, void* workspace, rnntOptions options);

/** Number of kernels launched by this library in this process since load (bench.py's gpu_launches).  Every kernel
 *  on the path is the library's own: it links no GEMM library. */
unsigned long long rnntb200_launch_count();

/** Per-kernel CUDA-event instrumentation for bench.py's attribution pass.  set_timing(1) clears the record
 *  list and enables recording (events on the launching stream around each hot kernel); set_timing(0)
 *  disables and clears.  After synchronising the stream, get_timing(i, &name, &ms) returns 1 and the i-th
 *  record, or 0 past the end.  Off by default; never enabled inside a timed benchmark region. */
void rnntb200_set_timing(int on);
int rnntb200_get_timing(int index, const char** name, float* ms);

/** Build info string: "rnnt_b200 <version> sm_90a wgmma=<0|1>". */
const char* rnntb200_build_info();

#ifdef __cplusplus
}
#endif
