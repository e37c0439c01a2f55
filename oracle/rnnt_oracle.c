/*
 * rnnt_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C restatement of the reference RNN-T loss hot path (joint network forward,
 * log-softmax, transducer alpha/beta dynamic program, gradients), used only as the
 * parity checker by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg.
 * The product path (rnnt_speech_recognition_b200/csrc) never links or calls it.
 *
 * Pinning: the float instantiation is checked against (i) the reference's own
 * known-answer tests (warp-transducer/tests/test_cpu.cpp:12-179, tests/test_gpu.cu:96-224,
 * pytorch_binding/test/test.py:51-160) and (ii) the reference library itself built into
 * oracle/_ref/ (see oracle/Makefile), or its stored outputs (tests/golden/ref_cases.npz) -- tests/test_oracle.py.
 * The joint (Dense/tanh/add) has no pinned vectors anywhere in the reference
 * (TensorFlow 2.2 arithmetic, un-vendored): that part is "parity unpinned" and is
 * anchored on model.py:158-166 plus an fp64 torch-autograd cross-check.
 *
 * Build: gcc -O2 -fopenmp -fPIC -shared rnnt_oracle.c -o liboracle.so -lm
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define REAL float
#define FN(x) x##_f32
#include "rnnt_oracle_impl.inc"
#undef REAL
#undef FN

#define REAL double
#define FN(x) x##_f64
#include "rnnt_oracle_impl.inc"
#undef REAL
#undef FN

/* get_workspace_size -- rnnt_entrypoint.cpp:96-128 (pure function; restated so the
 * host-side workspace sizing of the product can be checked without a GPU). */
int oracle_get_workspace_size(int maxT, int maxU, int minibatch, int gpu, size_t* size_bytes, size_t dtype_size) {
    if (minibatch <= 0 || maxT <= 0 || maxU <= 0) return 2;
    size_t per = dtype_size * (size_t)maxT * maxU * 2;
    if (!gpu) per += dtype_size * (size_t)maxT * maxU * 2;
    else { per += dtype_size * (size_t)maxT * maxU; per += dtype_size * 2; }
    *size_bytes = per * (size_t)minibatch;
    return 0;
}
