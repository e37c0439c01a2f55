// joint_tc.cuh -- tensor-core (wgmma / TMA / mbarrier) path of the fused joint + loss: shared definitions (tile
// geometry, kernel parameters, tensor maps, workspace layout, small helper kernels) and the host-side orchestration
// (tc_forward / tc_backward).  The kernels themselves: joint_fwd.cuh (forward), joint_bwd.cuh (the two backward
// contractions).  Persistent CTAs loop over 128-cell lattice tiles (16 time steps x 8 label positions of one utterance);
// the (B,T,U,H) activation tensor of model.py:158-163 and the (B,T,U,V) logits of model.py:165-166 never exist in HBM.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <mutex>
#include <unordered_map>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <cstdlib>

#include "../../include/rnnt_b200.h"
#include "kernels_simt.cuh"
#include "ptx.cuh"
#include "timing.cuh"

namespace rb {

constexpr int TC_MAX_KB = 16;        // H <= 1024
constexpr size_t TC_SMEM_OPTIN = 232448;   // largest dynamic shared memory a block may opt in to (sm_90: 227 KB)
constexpr int TC_SMS = 132;               // SM count the split-K workspace is sized for (H100 SXM); launches query the device

struct TcGeom {
    int TT, UU, nTb, nUb;  // tile = TT x UU cells (TT*UU == 128); tiles per utterance
    int KB;
    bool ok;
};

// Tile shape: 16 time steps x 8 label positions.  Every tile re-reads its TT enc rows and UU pred rows (fp32, H wide)
// from L2, so a balanced shape minimises that stream (1 x 128 tiles would cost 330 KB per tile, 16 x 8 cost 61 KB).
inline TcGeom tc_geometry(int maxT, int maxU, int H, int V) {
    TcGeom g{};
    g.ok = false;
    if (H % 64 || V % 64 || H > 64 * TC_MAX_KB) return g;
    g.UU = 8;
    g.TT = 16;
    g.nTb = (maxT + g.TT - 1) / g.TT;
    g.nUb = (maxU + g.UU - 1) / g.UU;
    g.KB = H / 64;
    g.ok = true;
    return g;
}

// SM count of the CURRENT device (queried per call: the library may be used on several devices of one process)
inline int tc_num_sms() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
        n = TC_SMS;
    return n;
}

struct JointTcParams {
    const float* enc; const float* pred; const float* bias;
    const int* labels; const int* xlen; const int* ylen;
    int B, maxT, maxU, H, V, blank;
    int TT, UU, nTb, nUb, KB, stages;
    long long SK;
    int b0, nb;                 // utterance range of this launch
    const int* slot;            // tile -> compact row block of the kept arrays (valid tiles only); NULL = tile order
    float* lse; float* lpb; float* lpl;              // outputs (NULL: a recompute that only wants the kept activations)
    // MODE 2 (forward that KEEPS its activations): dl receives the softmax numerators 2^(y - ref) as bf16, one row of V
    // per lattice cell, gm the row's reference ref (log2 domain).
    __nv_bfloat16* dl;
    float* gm;
    Windows win;                // alignment-restricted loss: per-column frame windows (lo == NULL: none)
};
// THE validity rule of a TT x UU tile at (b, t0, u0), shared by tile_compact_kernel (slots) and decode_tile (forward):
// the tile intersects the utterance's T_b x U_b lattice and, with windows, some column u in [u0, min(u0 + UU, U_b)) has
// [lo, hi] meet [t0, t0 + TT).  Full windows (lo <= 0, hi >= T_b - 1) therefore rank the tiles exactly as no windows do.
__device__ __forceinline__ bool tile_valid(int b, int t0, int u0, int Tn, int Un, int TT, int UU, int maxU, const Windows& w) {
    if (!(t0 < Tn && u0 < Un)) return false;
    if (!w.lo) return true;
    const int u1 = min(u0 + UU, Un);
    for (int u = u0; u < u1; ++u) {
        const int lo = w.lo[(long long)b * maxU + u], hi = w.hi[(long long)b * maxU + u];
        if (lo <= hi && lo < t0 + TT && hi >= t0) return true;
    }
    return false;
}
struct TileInfo { int b, t0, u0, Tn, Un; bool valid; };
__device__ __forceinline__ TileInfo decode_tile(const JointTcParams& p, int tile) {
    TileInfo ti;
    const int per_utt = p.nTb * p.nUb;
    const int bl = tile / per_utt, rem = tile - bl * per_utt;
    ti.b = p.b0 + bl;
    ti.t0 = (rem / p.nUb) * p.TT;
    ti.u0 = (rem % p.nUb) * p.UU;
    ti.Tn = p.xlen[ti.b];
    ti.Un = p.ylen[ti.b] + 1;
    ti.valid = tile_valid(ti.b, ti.t0, ti.u0, ti.Tn, ti.Un, p.TT, p.UU, p.maxU, p.win);
    return ti;
}

// W (H,V) fp32 -> Wt (V,H) fp16 [B operand of the logits GEMM, K=h] and Wb (H,V) bf16 [B operand of dZ, K=v]
__global__ void __launch_bounds__(256) convert_w_kernel(const float* __restrict__ W, __nv_bfloat16* __restrict__ Wt,
                                                        __nv_bfloat16* __restrict__ Wb, int H, int V) {
    __shared__ float tile[32][33];
    const int v0 = blockIdx.x * 32, h0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
    for (int i = ty; i < 32; i += 8) {
        const int h = h0 + i, v = v0 + tx;
        const float w = (h < H && v < V) ? W[(size_t)h * V + v] : 0.f;
        tile[i][tx] = w;
        if (h < H && v < V) Wb[(size_t)h * V + v] = __float2bfloat16(w);
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
        const int v = v0 + i, h = h0 + tx;
        if (h < H && v < V) reinterpret_cast<__half*>(Wt)[(size_t)v * H + h] = __float2half_rn(tile[tx][i]);
    }
}

// slot[tile] = rank of the tile among the VALID tiles (tile_valid) of this launch (-1 for the others); *count = #valid.
// One block; a serial-over-chunks block scan is plenty for the <= ~1e5 tiles of a launch.
__global__ void __launch_bounds__(1024) tile_compact_kernel(const int* __restrict__ xlen, const int* __restrict__ ylen,
                                                            int b0, int ntiles, int nTb, int nUb, int TT, int UU,
                                                            int* __restrict__ slot, int* __restrict__ count,
                                                            int* __restrict__ tile_of_slot = nullptr,
                                                            int4* __restrict__ slot_meta = nullptr, int maxT = 0, int maxU = 0,
                                                            int max_slots = 0x7fffffff,
                                                            const Windows win = Windows{nullptr, nullptr}) {
    __shared__ int warp_sums[32];
    __shared__ int base;
    if (threadIdx.x == 0) base = 0;
    __syncthreads();
    const int per_utt = nTb * nUb, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int t0 = 0; t0 < ntiles; t0 += 1024) {
        const int tile = t0 + threadIdx.x;
        int v = 0;
        int4 meta = make_int4(0, 0, 1, 1);
        if (tile < ntiles) {
            const int bl = tile / per_utt, rem = tile - bl * per_utt, b = b0 + bl;
            const int tt = (rem / nUb) * TT, uu = (rem % nUb) * UU;
            v = tile_valid(b, tt, uu, xlen[b], ylen[b] + 1, TT, UU, maxU, win) ? 1 : 0;
            // what the kernels that walk the compact slots need of a tile, so that none of them divides: first enc / pred row
            // (in rows of H floats) and how many of the tile's TT / UU rows exist in the padded arrays
            meta = make_int4(b * maxT + tt, b * maxU + uu, min(TT, maxT - tt), min(UU, maxU - uu));
        }
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int w = warp_sums[lane], wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int n = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += n; }
            warp_sums[lane] = wi - w;   // exclusive prefix of the warp totals
        }
        __syncthreads();
        const int excl = base + warp_sums[warp] + incl - v;
        if (tile < ntiles) {
            // a valid tile beyond the row blocks the workspace holds (the caller's valid_tile_bound was too small) gets no slot:
            // nothing is stored for it, the overflow word is raised and the forward call poisons the costs
            const bool fits = excl < max_slots;
            slot[tile] = (v && fits) ? excl : -1;
            if (v && fits && tile_of_slot) tile_of_slot[excl] = tile;
            if (v && fits && slot_meta) slot_meta[excl] = meta;
        }
        __syncthreads();
        if (threadIdx.x == 1023) base = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        count[0] = min(base, max_slots);
        count[1] = base > max_slots ? base : 0;        // overflow word: the number of valid tiles found
        if (base > max_slots)
            printf("rnnt_b200: %d lattice tiles are valid but rnntb200JointDesc.valid_tile_bound promised at most %d -- results are invalid\n",
                   base, max_slots);
    }
}
// out[i] = sum_k part[k][i] over `nplanes` planes of `n4` float4 each
__global__ void __launch_bounds__(256) sum_planes_kernel(const float4* __restrict__ part, int nplanes, size_t n4,
                                                         float4* __restrict__ out) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
        for (int k = 0; k < nplanes; ++k) {
            const float4 v = part[(size_t)k * n4 + i];
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        out[i] = acc;
    }
}
// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
    return fn;
}
// 2-D row-major bf16 matrix [rows x cols] (cols contiguous, rows `ld` elements apart: cols when 0), box [box_rows x 64
// cols], SWIZZLE_128B
inline bool make_tmap_bf16(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows,
                           uint32_t box_cols = 64, uint64_t ld = 0) {
    PFN_encodeTiled fn = get_encode_fn();
    if (!fn) return false;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {(ld ? ld : cols) * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    return fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// 2-D row-major fp32 matrix [rows x cols], box [box_rows x 128 cols] stored densely (no swizzle); out-of-range reads as 0
inline bool make_tmap_f32(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    PFN_encodeTiled fn = get_encode_fn();
    if (!fn) return false;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {cols * 4};
    cuuint32_t box[2] = {128, box_rows};
    cuuint32_t estr[2] = {1, 1};
    return fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Workspace of the tensor-core path (a pure function of the descriptor).  The kept arrays (numerators + maxima) are
// laid out per 128-row tile; the batch is processed in utterance chunks that keep them under ~16 GiB.
struct TcScratch {
    __nv_bfloat16 *Wt, *Wb;                 // W^T (V,H) fp16 [forward B operand, 16-bit storage] and W (H,V) bf16 [dZ B operand]
    __nv_bfloat16* dl;                      // (rows_chunk, V) bf16 softmax numerators E = 2^(y - ref_row)
    float* gm;                              // (rows_chunk) fp32 reference of each row's numerators (log2 domain)
    int* slot;                              // tile -> compact row block (-1: outside the valid lattice), per chunk
    int* tile_of_slot;                      // compact row block -> tile
    int4* slot_meta;                        // compact row block -> {first enc row, first pred row, #t rows, #u rows} (tile_compact_kernel)
    int* count;                             // number of valid tiles of the chunk
    float* ppl;                             // (nTb, bchunk, maxU, H) fp32 partial planes of d_pred (bwd_dz_kernel)
    float* dWp;                             // (S_max, H, V) fp32 split-K planes of dW (bwd_dw_kernel)
    float* dbp;                             // (S_max, V) planes of db
    float* rowscale;                        // (rows_chunk) per-row scale of the logit gradients (row_scale_kernel)
    __nv_bfloat16* zs;                      // (rows_chunk, zs_ld) bf16 dW operand [rs * z, rs] (bwd_dz_kernel)
    int zs_ld;                              // H + 64: rows start on 128-byte lines
    int bchunk;                             // utterances per chunk
    size_t rows_chunk;                      // bchunk * tiles_per_utt * 128
    size_t bytes;
};
// bytes of kept activations per utterance chunk: 16 GiB (RNNTB200_CHUNK_MB overrides it for the tests of the
// multi-chunk backward; read once per process, so the workspace size stays a pure function of the descriptor)
inline size_t tc_chunk_budget() {
    static size_t v = 0;
    if (!v) { const char* e = getenv("RNNTB200_CHUNK_MB"); v = e && atoll(e) > 0 ? (size_t)atoll(e) << 20 : (size_t)16 << 30; }
    return v;
}
inline rnntStatus_t tc_unsupported(const rnntb200JointDesc& d) {
    fprintf(stderr,
            "rnnt_b200: RNNTB200_BF16_TC needs H %% 64 == 0, V %% 64 == 0 and 64 <= H <= 768 (got H=%d V=%d); "
            "use RNNTB200_FP32_EXACT\n", d.H, d.V);
    return RNNT_STATUS_INVALID_VALUE;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE property of a kernel: set it once per (device, kernel),
// thread-safe (the library may be driven from several host threads / several devices of one process).
inline bool tc_smem_optin(const void* func, size_t bytes = TC_SMEM_OPTIN) {
    static std::mutex mu;
    static std::unordered_map<unsigned long long, bool> done;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return false;
    const unsigned long long key = (unsigned long long)reinterpret_cast<uintptr_t>(func) * 64ull + (unsigned long long)dev;
    std::lock_guard<std::mutex> lk(mu);
    auto it = done.find(key);
    if (it != done.end()) return true;
    if (cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) != cudaSuccess) {
        cudaGetLastError();         // reported by the caller's status: not left pending for the next call's launch check
        return false;
    }
    done[key] = true;
    return true;
}

}  // namespace rb

#include "joint_fwd.cuh"
#include "joint_bwd.cuh"

namespace rb {

inline TcScratch tc_scratch_layout(const rnntb200JointDesc& d, void* base) {
    TcScratch s{};
    const TcGeom g = tc_geometry(d.maxT, d.maxU, d.H, d.V);
    const DwGeom wg = dw_geometry(d.H, d.V);
    const size_t rows_utt = (size_t)g.nTb * g.nUb * 128;
    const size_t per_row = (size_t)d.V * 2 + 8;
    size_t bc = tc_chunk_budget() / (rows_utt * per_row);
    if (bc < 1) bc = 1;
    if (bc > (size_t)d.B) bc = d.B;
    s.bchunk = (int)bc;
    s.rows_chunk = bc * rows_utt;
    // The kept arrays are indexed by COMPACT slots (valid tiles only), but how many tiles are valid is known to the device
    // alone, so the default sizes them for every tile of the padded (maxT, maxU) lattice and chunks the batch.  A caller
    // that knows its lengths on the host can promise an upper bound: the whole batch is then ONE chunk of that many row
    // blocks, as long as they fit in 56 GiB (an 80 GB device also holds the inputs, the loss planes and the gradients).
    if (d.valid_tile_bound > 0 && bc < (size_t)d.B) {
        const size_t tiles = (size_t)d.valid_tile_bound < (size_t)d.B * g.nTb * g.nUb ? (size_t)d.valid_tile_bound : (size_t)d.B * g.nTb * g.nUb;
        if (tiles * 128 * per_row <= ((size_t)56 << 30)) { bc = d.B; s.bchunk = d.B; s.rows_chunk = tiles * 128; }
    }
    char* p = static_cast<char*>(base);
    auto take = [&](size_t n) { char* r = p; p += (n + 255) / 256 * 256; return r; };
    s.Wt = reinterpret_cast<__nv_bfloat16*>(take((size_t)d.V * d.H * 2));
    s.Wb = reinterpret_cast<__nv_bfloat16*>(take((size_t)d.V * d.H * 2));
    s.dl = reinterpret_cast<__nv_bfloat16*>(take(s.rows_chunk * d.V * 2));
    s.gm = reinterpret_cast<float*>(take(s.rows_chunk * 4));
    s.slot = reinterpret_cast<int*>(take((size_t)bc * g.nTb * g.nUb * 4));
    s.tile_of_slot = reinterpret_cast<int*>(take((size_t)bc * g.nTb * g.nUb * 4));
    s.slot_meta = reinterpret_cast<int4*>(take((size_t)bc * g.nTb * g.nUb * 16));
    s.count = reinterpret_cast<int*>(take(256));
    s.ppl = reinterpret_cast<float*>(take((size_t)g.nTb * bc * d.maxU * d.H * 4));
    s.dWp = reinterpret_cast<float*>(take((size_t)wg.S * d.H * d.V * 4));
    s.dbp = reinterpret_cast<float*>(take((size_t)wg.S * d.V * 4));
    s.rowscale = reinterpret_cast<float*>(take(s.rows_chunk * 4));
    // the dW operand is not part of the chunk plan above: the plan (and with it how many times the dW planes are
    // accumulated) sizes the kept numerators alone, and zs adds rows_chunk * (H + 64) * 2 bytes on top of it.  Rows
    // start on 128-byte lines, so that every 64-column box row the dZ kernel stores and the dW kernel loads is one whole
    // line (with a row stride of H + 8, merely 16-byte aligned, the C3 step was 2 ms slower).
    s.zs_ld = d.H + 64;
    s.zs = reinterpret_cast<__nv_bfloat16*>(take(s.rows_chunk * s.zs_ld * 2));
    s.bytes = (size_t)(p - static_cast<char*>(base));
    return s;
}

inline bool tc_supported(const rnntb200JointDesc& d) {
    return tc_geometry(d.maxT, d.maxU, d.H, d.V).ok && d.H <= 768 && fwd_geometry(d.H, d.V).ok && dz_geometry(d.H).ok;
}
inline size_t tc_scratch_bytes(const rnntb200JointDesc& d) {
    if (!tc_supported(d)) return 0;
    return tc_scratch_layout(d, nullptr).bytes;
}

// keep_activations is honoured when the whole batch is one workspace chunk (RNNTB200_KEEP=0 turns it off for A/B
// measurements); otherwise the backward re-runs the keeping forward chunk by chunk.
inline bool tc_keep(const rnntb200JointDesc& d, const TcScratch& sc) {
    static int env = -1;
    if (env < 0) { const char* e = getenv("RNNTB200_KEEP"); env = e ? atoi(e) : 1; }
    return d.keep_activations && env && sc.bchunk >= d.B;
}

// the forward kernel over utterances [b0, b0+nb); KEEP: rank the chunk's valid tiles on the device (nothing is read
// back) and leave numerators + references in the workspace
template <bool KEEP>
inline rnntStatus_t tc_run_forward(const rnntb200JointDesc& d, const TcGeom& g, const TcScratch& sc, const float* enc,
                                   const float* pred, const float* bias, const int* labels, const int* ylen,
                                   const int* xlen, float* lse, float* lpb, float* lpl, int b0, int nb, cudaStream_t s,
                                   unsigned* launches, const Windows& win) {
    const FwdGeom fg = fwd_geometry(d.H, d.V);
    JointTcParams p{};
    p.enc = enc; p.pred = pred; p.bias = bias; p.labels = labels; p.xlen = xlen; p.ylen = ylen;
    p.B = d.B; p.maxT = d.maxT; p.maxU = d.maxU; p.H = d.H; p.V = d.V; p.blank = d.blank_label;
    p.TT = g.TT; p.UU = g.UU; p.nTb = g.nTb; p.nUb = g.nUb; p.KB = g.KB;
    p.SK = (long long)(d.maxT + d.maxU - 1) * d.maxU;
    p.b0 = b0; p.nb = nb;
    p.lse = lse; p.lpb = lpb; p.lpl = lpl;
    p.stages = fg.stages;
    p.win = win;
    if (KEEP) {
        const int ntiles = nb * g.nTb * g.nUb;
        tile_compact_kernel<<<1, 1024, 0, s>>>(xlen, ylen, b0, ntiles, g.nTb, g.nUb, g.TT, g.UU, sc.slot, sc.count, sc.tile_of_slot, sc.slot_meta,
                                             d.maxT, d.maxU, (int)(sc.rows_chunk / 128), win);
        *launches += 1;
        p.slot = sc.slot; p.dl = sc.dl; p.gm = sc.gm;
    }
    CUtensorMap tm;
    if (!make_tmap_bf16(&tm, sc.Wt, d.V, d.H, FWD_NC)) {
        fprintf(stderr, "rnnt_b200: cuTensorMapEncodeTiled failed\n");
        return RNNT_STATUS_EXECUTION_FAILED;
    }
    *launches += 1;
    return fwd_launch<KEEP ? 2 : 0>(fg, tm, p, s);
}

inline rnntStatus_t tc_forward(const rnntb200JointDesc& d, void* scratch, const float* enc, const float* pred,
                               const float* W, const float* bias, const int* labels, const int* ylen,
                               const int* xlen, float* lse, float* lpb, float* lpl, cudaStream_t s,
                               unsigned* launches, const Windows& win) {
    if (!tc_supported(d)) return tc_unsupported(d);
    const TcGeom g = tc_geometry(d.maxT, d.maxU, d.H, d.V);
    TcScratch sc = tc_scratch_layout(d, scratch);
    convert_w_kernel<<<dim3((d.V + 31) / 32, (d.H + 31) / 32), 256, 0, s>>>(W, sc.Wt, sc.Wb, d.H, d.V);
    *launches += 1;
    if (tc_keep(d, sc))
        return tc_run_forward<true>(d, g, sc, enc, pred, bias, labels, ylen, xlen, lse, lpb, lpl, 0, d.B, s, launches, win);
    return tc_run_forward<false>(d, g, sc, enc, pred, bias, labels, ylen, xlen, lse, lpb, lpl, 0, d.B, s, launches, win);
}

// The valid_tile_bound promise of a call that keeps nothing (alignment): when a bound is given and the batch is one
// workspace chunk, the tiles are counted as the keeping forward counts them.  Returns the overflow word (nonzero:
// the promise is broken) or nullptr when there is nothing to check.
inline const int* tc_check_tile_bound(const rnntb200JointDesc& d, void* scratch, const int* ylen, const int* xlen,
                                      cudaStream_t s, unsigned* launches) {
    if (d.valid_tile_bound <= 0 || !tc_supported(d)) return nullptr;
    const TcScratch sc = tc_scratch_layout(d, scratch);
    if (sc.bchunk < d.B) return nullptr;
    const TcGeom g = tc_geometry(d.maxT, d.maxU, d.H, d.V);
    tile_compact_kernel<<<1, 1024, 0, s>>>(xlen, ylen, 0, d.B * g.nTb * g.nUb, g.nTb, g.nUb, g.TT, g.UU, sc.slot, sc.count,
                                           nullptr, nullptr, d.maxT, d.maxU, (int)(sc.rows_chunk / 128));
    *launches += 1;
    return sc.count + 1;
}

struct LossPlanes { const float *lse, *lpb, *lpl, *alphas, *betas, *llf; };   // outputs of the forward + alpha/beta (loss workspace)

// Backward (SURVEY 8 a19) with the library's own wgmma kernels (joint_bwd.cuh).  Per utterance chunk: (a keeping forward
// of the chunk unless the forward call already kept the whole batch) -> row_scale_kernel -> bwd_dz_kernel -> d_pred plane
// sum -> bwd_dw_kernel; after the last chunk the split-K planes of dW / db are summed.  Stream-ordered, no host
// synchronisation, no library calls.  Windows reach the backward through the slots (tiles outside them have none),
// row_scale_kernel (rows outside them get rs = 0) and nothing else.  FastEmit lives entirely in row_scale_kernel (every chunk, keep or recompute): the
// GEMM kernels consume E' as they always do.
inline rnntStatus_t tc_backward(const rnntb200JointDesc& d, void* scratch, const float* enc, const float* pred,
                                const float* bias, const int* labels, const int* ylen, const int* xlen,
                                const LossPlanes& lp, const float* grad_costs, float* d_enc, float* d_pred, float* dW,
                                float* db, cudaStream_t s, unsigned* launches, float fastemit_lambda, const Windows& win) {
    if (!tc_supported(d)) return tc_unsupported(d);
    const TcGeom g = tc_geometry(d.maxT, d.maxU, d.H, d.V);
    const DzGeom zg = dz_geometry(d.H);
    const DwGeom wg = dw_geometry(d.H, d.V);
    TcScratch sc = tc_scratch_layout(d, scratch);   // Wt / Wb were produced by the forward call
    const bool kept = tc_keep(d, sc);
    if (!tc_smem_optin(reinterpret_cast<const void*>(bwd_dz_kernel)) || !tc_smem_optin(reinterpret_cast<const void*>(bwd_dw_kernel)))
        return RNNT_STATUS_EXECUTION_FAILED;
    if (cudaMemsetAsync(sc.dWp, 0, sizeof(float) * (size_t)wg.S * d.H * d.V, s) != cudaSuccess ||
        cudaMemsetAsync(sc.dbp, 0, sizeof(float) * (size_t)wg.S * d.V, s) != cudaSuccess)
        return RNNT_STATUS_MEMOPS_FAILED;
    // the dW operand is stored through a map H columns wide (column H, the row scale, is written directly) and loaded
    // through one H + 1 wide, so that the columns past H of the last row block read as zeros
    CUtensorMap tm_e128, tm_e64, tm_w, tm_enc, tm_pred, tm_zs_st, tm_zs_ld;
    if (!make_tmap_bf16(&tm_e128, sc.dl, sc.rows_chunk, d.V, 128) || !make_tmap_bf16(&tm_e64, sc.dl, sc.rows_chunk, d.V, 64) ||
        !make_tmap_bf16(&tm_w, sc.Wb, d.H, d.V, DZ_NC) ||
        !make_tmap_bf16(&tm_zs_st, sc.zs, sc.rows_chunk, d.H, 128, 64, sc.zs_ld) ||
        !make_tmap_bf16(&tm_zs_ld, sc.zs, sc.rows_chunk, d.H + 1, 64, 64, sc.zs_ld) ||
        !make_tmap_f32(&tm_enc, enc, (uint64_t)d.B * d.maxT, d.H, BW_TT) || !make_tmap_f32(&tm_pred, pred, (uint64_t)d.B * d.maxU, d.H, BW_UU)) {
        fprintf(stderr, "rnnt_b200: cuTensorMapEncodeTiled failed\n");
        return RNNT_STATUS_EXECUTION_FAILED;
    }
    const int sms = tc_num_sms();
    for (int b0 = 0; b0 < d.B; b0 += sc.bchunk) {
        const int nb = (d.B - b0 < sc.bchunk) ? d.B - b0 : sc.bchunk;
        if (!kept) {
            rnntStatus_t st = tc_run_forward<true>(d, g, sc, enc, pred, bias, labels, ylen, xlen, nullptr, nullptr, nullptr, b0, nb, s, launches, win);
            if (st) return st;
        }
        {   // per-row scales of this chunk (row order of the kept arrays) + the two special columns of every row
            ScopedTimer tmr("row_scale_kernel", s);
            row_scale_kernel<<<(unsigned)(((size_t)nb * g.nTb * g.nUb * 128 + 255) / 256), 256, 0, s>>>(
                sc.tile_of_slot, sc.count, b0, g.nTb, g.nUb, xlen, ylen, labels, d.blank_label, d.maxT, d.maxU,
                (long long)(d.maxT + d.maxU - 1) * d.maxU, lp.lse, lp.lpb, lp.lpl, lp.alphas, lp.betas, lp.llf, grad_costs, sc.gm,
                d.V, reinterpret_cast<unsigned short*>(sc.dl), sc.rowscale, fastemit_lambda, win);
            *launches += 1;
        }
        BwdParams p{};
        p.enc = enc; p.pred = pred; p.xlen = xlen; p.ylen = ylen;
        p.maxT = d.maxT; p.maxU = d.maxU; p.H = d.H; p.V = d.V;
        p.nTb = g.nTb; p.nUb = g.nUb; p.b0 = b0; p.nb = nb;
        p.slot = sc.slot; p.slot_meta = sc.slot_meta; p.count = sc.count; p.rowscale = sc.rowscale;
        p.dz_stages = zg.stages; p.d_enc = d_enc; p.ppred = sc.ppl; p.zs = sc.zs; p.zs_ld = sc.zs_ld;
        p.nVT = wg.nCT; p.nHB = wg.nHB; p.S = wg.S; p.dWp = sc.dWp; p.dbp = sc.dbp;
        // rows of d_enc whose t-block lies outside the utterance are never visited by the dZ kernel (a t-block inside it
        // without a valid tile is: its rows are stored as the zeros they are)
        if (cudaMemsetAsync(d_enc + (size_t)b0 * d.maxT * d.H, 0, sizeof(float) * (size_t)nb * d.maxT * d.H, s) != cudaSuccess)
            return RNNT_STATUS_MEMOPS_FAILED;
        {
            const int nruns = nb * g.nTb;
            ScopedTimer tmr("bwd_dz_kernel", s);
            bwd_dz_kernel<<<nruns < sms ? nruns : sms, BWD_THREADS, zg.smem_bytes, s>>>(tm_e128, tm_w, tm_enc, tm_pred, tm_zs_st, p);
        }
        {
            const size_t n4 = (size_t)nb * d.maxU * d.H / 4;
            ScopedTimer tmr("sum_pred_planes_kernel", s);
            sum_pred_planes_kernel<<<(unsigned)((n4 + 255) / 256 < 4096 ? (n4 + 255) / 256 : 4096), 256, 0, s>>>(
                reinterpret_cast<const float4*>(sc.ppl), sc.slot, g.nTb, g.nUb, xlen, ylen, b0, nb, d.maxU, d.H / 4,
                reinterpret_cast<float4*>(d_pred));
        }
        {
            ScopedTimer tmr("bwd_dw_kernel", s);
            bwd_dw_kernel<<<wg.nCT * wg.nHB * wg.S, DW_THREADS, wg.smem_bytes, s>>>(tm_e64, tm_zs_ld, p);
        }
        *launches += 3;
        if (cudaGetLastError() != cudaSuccess) return RNNT_STATUS_EXECUTION_FAILED;
    }
    {
        ScopedTimer tmr("sum_planes_kernel", s);
        const size_t nw4 = (size_t)d.H * d.V / 4, nb4 = (size_t)d.V / 4;
        sum_planes_kernel<<<(unsigned)((nw4 + 255) / 256 < 4096 ? (nw4 + 255) / 256 : 4096), 256, 0, s>>>(
            reinterpret_cast<const float4*>(sc.dWp), wg.S, nw4, reinterpret_cast<float4*>(dW));
        sum_planes_kernel<<<(unsigned)((nb4 + 255) / 256), 256, 0, s>>>(reinterpret_cast<const float4*>(sc.dbp), wg.S, nb4,
                                                                       reinterpret_cast<float4*>(db));
    }
    *launches += 2;
    return cudaGetLastError() == cudaSuccess ? RNNT_STATUS_SUCCESS : RNNT_STATUS_EXECUTION_FAILED;
}
}  // namespace rb
