// lep_common.cuh -- shared device-side definitions for the Lepton coder kernels.
//
// This is a from-scratch sm_90a design of dropbox/lepton's arithmetic-coding hot path.  What is kept from
// the reference is the *bitstream semantics* (so that .lep bytes are identical); the data layout, the work
// decomposition (one warp per thread-segment, lane-parallel symbolisation of two blocks at a time, batched model
// update, one range-coder thread per segment) and the probability-table representation are new.
//
// Reference semantics cited below are relative to /root/reference.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace lepb200 {

constexpr unsigned FULL = 0xffffffffu;

// Cache hints for data that streams through (build-time option LEPB200_STREAM_HINTS=1; results are unchanged, only the
// eviction priority in L1 / L2): the coefficient planes, the token streams and the model zero fill add up to several
// times the 50 MB L2 per launch, while the lines that ARE reused -- the touched part of each resident model, ~49 KB per
// segment -- are what the kernels wait for.  LEP_LD_LAST = last use of a line (the row above, read a second time),
// LEP_ST_STREAM = written once and read by a later kernel.  Off by default until it is measured on the GPU.
// (macros, not functions: a pointer passed through a function parameter loses its __restrict__ and the default build
// must keep the SASS that was validated on the GPU)
#if defined(LEPB200_STREAM_HINTS) && LEPB200_STREAM_HINTS && !defined(LEPB200_EMU)
#define LEP_LD_LAST(p, i) __ldcs((p) + (i))
#define LEP_ST_STREAM(p, i, v) __stcs((p) + (i), (v))
#else
#define LEP_LD_LAST(p, i) p[i]
#define LEP_ST_STREAM(p, i, v) p[i] = v
#endif

// ------------------------------------------------------------------------------------------------------
// Probability model layout.
//
// The reference keeps 721 564 three-byte Branch objects (counts[2] + cached probability, 2.1 MB) per
// thread-segment (src/vp8/model/model.hh:60-127, branch.hh:11-128) and re-initialises them to (1,1,128)
// with a 2.1 MB memset per segment.  Here a branch is ONE 16-bit word  (c0-1) | (c1-1)<<8 :
//   * all-zero memory IS the identity prior, so a segment's model is reset by a plain zero fill;
//   * the probability is recomputed from the counts on use,  p = (c0<<8)/(c0+c1)  (branch.hh:108-120),
//     off the range coder's serial dependency chain;
//   * the one state whose cached probability is not a function of its counts -- (1,255) reached through
//     the "neverseen" overflow, p = 0 (branch.hh:87-90) -- is encoded with the otherwise unused low byte 0xff.
// Exponent contexts are padded from 11 to 16 entries so that one context's unary chain is exactly one
// 32-byte sector.  Only the bins the grammar can reach are allocated (10 of 26 nz-count bins).
// ------------------------------------------------------------------------------------------------------
constexpr uint32_t M_NZ7 = 0;                                        // [2][10][6][32]
constexpr uint32_t M_NZE = M_NZ7 + 2 * 10 * 6 * 32;                  // [2 kinds][2][8][8][3][4]  (kind 0 = 8x1 horizontal, 1 = 1x8 vertical)
constexpr uint32_t M_RESN = M_NZE + 2 * 2 * 8 * 8 * 3 * 4;           // [2][64][10][16]  (10 used)
constexpr uint32_t M_RESDC = M_RESN + 2 * 64 * 10 * 16;              // [12][16]
constexpr uint32_t M_EXP7 = M_RESDC + 12 * 16;                       // [2][10][49][12][16]
constexpr uint32_t M_EXPX = M_EXP7 + 2 * 10 * 49 * 12 * 16;          // [2][8][15][12][16]
constexpr uint32_t M_EXPDC = M_EXPX + 2 * 8 * 15 * 12 * 16;          // [12][17][16]
constexpr uint32_t M_SIGN = M_EXPDC + 12 * 17 * 16;                  // [2][4][12] (+pad)
constexpr uint32_t M_THR = M_SIGN + 128;                             // [2][256][8][128]
constexpr uint32_t M_TOTAL = M_THR + 2 * 256 * 8 * 128;              // u16 entries
static_assert(M_TOTAL < (1u << 20), "branch index must fit in 20 bits");
static_assert((M_TOTAL % 8) == 0, "model zero fill uses 16-byte stores");
constexpr size_t MODEL_BYTES = size_t(M_TOTAL) * 2;

__host__ __device__ inline uint32_t m_nz7(int ci, int bin, int idx, int prefix) { return M_NZ7 + (((ci * 10 + bin) * 6 + idx) << 5) + prefix; }
__host__ __device__ inline uint32_t m_nze(int vertical, int ci, int eob, int nzb, int idx, int prefix) {
    return M_NZE + (((((vertical * 2 + ci) * 8 + eob) * 8 + nzb) * 3 + idx) << 2) + prefix;
}
// (a position-innermost variant of the three big tables was measured slower for both kernel A and the decode kernel, and dropped)
__host__ __device__ inline uint32_t m_resn(int ci, int coord, int bin) { return M_RESN + (((ci * 64 + coord) * 10 + bin) << 4); }
__host__ __device__ inline uint32_t m_exp7(int ci, int bin, int zz, int bsr) { return M_EXP7 + ((((ci * 10 + bin) * 49 + zz) * 12 + bsr) << 4); }
__host__ __device__ inline uint32_t m_expx(int ci, int ne, int zig15, int bsr) { return M_EXPX + ((((ci * 8 + ne) * 15 + zig15) * 12 + bsr) << 4); }
__host__ __device__ inline uint32_t m_resdc(int lenmxm) { return M_RESDC + (lenmxm << 4); }
__host__ __device__ inline uint32_t m_expdc(int a, int b) { return M_EXPDC + ((a * 17 + b) << 4); }
__host__ __device__ inline uint32_t m_sign(int ci, int a, int b) { return M_SIGN + (ci * 4 + a) * 12 + b; }
__host__ __device__ inline uint32_t m_thr(int ci, int ctx, int len) { return M_THR + (((ci * 256 + ctx) * 8 + len) << 7); }

// ------------------------------------------------------------------------------------------------------
// Small constant tables (reference: src/vp8/util/aligned_block.hh:32-55, src/vp8/model/jpeg_meta.hh:72-170 row 9).
// ------------------------------------------------------------------------------------------------------
static __constant__ uint8_t c_aligned_to_raster[64] = {
    9, 10, 17, 25, 18, 11, 12, 19, 26, 33, 41, 34, 27, 20, 13, 14, 21, 28, 35, 42, 49, 57, 50, 43, 36,
    29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63,
    0, 1, 2, 3, 4, 5, 6, 7, 8, 16, 24, 32, 40, 48, 56};
static __constant__ uint8_t c_nonzero_to_bin[50] = {
    0, 1, 2, 3, 4, 4, 5, 5, 5, 6, 6, 6, 6, 7, 7, 7, 7, 7, 7, 7, 7, 8, 8, 8, 8,
    8, 8, 8, 8, 8, 8, 8, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9};

// ------------------------------------------------------------------------------------------------------
// Job descriptors (device memory, written by the host side in lep_capi.cu).
// ------------------------------------------------------------------------------------------------------
struct ImageDesc {
    int32_t ncmp, mcuv;
    int32_t bch[3], bcv[3];          // blocks per row / rows of the allocated plane (componentInfo.bch/.bcv)
    int32_t trunc_bcv[3];            // rows actually coded   (UncompressedComponents::get_max_coded_heights)
    int32_t trunc_bc[3];             // blocks actually coded (component_size_in_blocks)
    int32_t mult[3];                 // bcv / mcuv: component rows per MCU row (lepton_codec.hh:55-57)
    int32_t pad_;
    unsigned long long plane[3];     // device address of the component's coefficient plane (AlignedBlock order)
    uint16_t q[3][64];               // quantisation table, raster order (model.hh:248-250)
    int32_t icos_x[3][64];           // model.hh:254
    int32_t icos_y[3][64];           // model.hh:255
    uint8_t min_thr[3][64];          // model.hh:277-289
};

struct SegDesc {
    int32_t image;                   // index into ImageDesc[]
    int32_t min_y, max_y, is_last;   // luma rows [min_y, max_y); last segment ignores max_y (vp8_encoder.cc:277-279)
    unsigned long long stream;       // device address of this segment's bool-coder byte stream
    uint32_t cap;                    // encode: capacity of stream; decode: length of stream
    uint32_t len;                    // encode: bytes produced
    int32_t status;                  // reference ExitCode value (0 ok, 6 COEFFICIENT_OUT_OF_RANGE, 7 STREAM_INCONSISTENT, ...)
    uint32_t ndecisions_lo, ndecisions_hi;
    uint32_t ntok;                   // encode: (probability, bit) tokens produced by kernel A
    unsigned long long tokens;       // encode: device address of the segment's token stream (uint16 each)
    uint32_t tok_cap;
    uint32_t total_shift;            // encode, parallel range coder: bits the coder shifted out over the whole segment (incl. marker and stop bits)
    unsigned long long digits;       // encode, parallel range coder: offset of the segment's 16-bit digits in the digit arena
    unsigned long long ovf;          // encode, parallel range coder: 1 + offset of the segment's stream in the overflow arena when
                                     // the stream does not fit `cap` (lep_digit_offsets_kernel), 0 when it stays where it is
};

enum : int32_t { ST_OK = 0, ST_ASSERT = 1, ST_COEF_RANGE = 6, ST_STREAM_INCONSISTENT = 7, ST_OUT_OVERFLOW = 100 };

// ------------------------------------------------------------------------------------------------------
// Branch word helpers.
// ------------------------------------------------------------------------------------------------------
// Exact floor((c0<<8)/(c0+c1)) via a 512-entry reciprocal table r[s] = ceil(2^32/s) in shared memory:
// __umulhi(n, r[s]) == n/s for all n < 2^16, s <= 510 (error < 2^-16 < 1/510).
__device__ __forceinline__ uint32_t branch_prob(uint32_t w, const uint32_t* __restrict__ s_rcp) {
    uint32_t lo = w & 0xff, hi = (w >> 8) & 0xff;
    uint32_t c0 = lo + 1, s = lo + hi + 2;
    uint32_t p = __umulhi(c0 << 8, s_rcp[s]);
    return lo == 0xff ? 0u : p;      // special state (c0=1,c1=255,p=0)
}
// Branch::record_obs_and_update (branch.hh:82-100) on the packed word.
__device__ __forceinline__ uint32_t branch_update(uint32_t w, uint32_t obs) {
    uint32_t lo = w & 0xff, hi = (w >> 8) & 0xff;
    bool special = lo == 0xff;                       // represents c0 == 1
    uint32_t c0 = special ? 1u : lo + 1, c1 = hi + 1;
    if (obs) {
        if (c1 == 255) {                             // overflow of the true count
            if (c0 == 1) return 0xfeffu;             // neverseen: stays (1,255), p = 0  -> special encoding
            c0 = (1 + c0) >> 1; c1 = 129;
        } else {
            c1 += 1;
        }
    } else {
        if (c0 == 255) {
            if (c1 == 1) return 0x00feu;             // (255,1), p = 255 == (255<<8)/256: representable normally
            c0 = 129; c1 = (1 + c1) >> 1;
        } else {
            c0 += 1;
        }
    }
    return (c0 - 1) | ((c1 - 1) << 8);
}

__device__ __forceinline__ int bitlen(uint32_t v) { return 32 - __clz(v); }
__device__ __forceinline__ int iabs(int v) { return v < 0 ? -v : v; }
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// lo/hi halves of a packed pair of int16 coefficients (aligned indices 2*lane, 2*lane+1)
__device__ __forceinline__ int h_lo(uint32_t w) { return (int)(int16_t)(w & 0xffff); }
__device__ __forceinline__ int h_hi(uint32_t w) { return (int)(int16_t)(w >> 16); }

// compute_aavrg_vec (model.hh:895-924): 16-bit lane arithmetic
__device__ __forceinline__ int aavrg16(int l, int a, int al, bool has_left, bool has_above) {
    if (!has_left && !has_above) return 0;
    uint32_t L = (uint32_t)iabs(l) & 0xffff, A = (uint32_t)iabs(a) & 0xffff;
    if (has_left && !has_above) return (int)(int16_t)L;
    if (!has_left) return (int)(int16_t)A;
    uint32_t t = ((L + A) * 13u + (((uint32_t)iabs(al) & 0xffff) * 6u)) & 0xffff;
    return (int)(t >> 5);
}

// LeptonCodec_row_spec_from_index (src/lepton/lepton_codec.hh:41-100)
struct RowSpec { int luma_y, component, curr_y; bool skip, done; };
__device__ inline RowSpec row_spec_from_index(uint32_t idx, const ImageDesc& g) {
    uint32_t m0 = g.mult[0], m1 = g.ncmp > 1 ? g.mult[1] : 0, m2 = g.ncmp > 2 ? g.mult[2] : 0;
    uint32_t mm = m0 + m1 + m2;
    uint32_t mcu_row = idx / mm, place = idx - mcu_row * mm;
    RowSpec r;
    r.luma_y = (int)(mcu_row * m0); r.skip = false; r.done = false;
    int i; uint32_t mi;
    if (place < m2) { i = 2; mi = m2; }
    else if (place - m2 < m1) { i = 1; mi = m1; place -= m2; }
    else { i = 0; mi = m0; place -= m2 + m1; }
    r.component = i;
    r.curr_y = (int)(mcu_row * mi + place);
    if (r.curr_y >= g.trunc_bcv[i]) {          // trunc_bcv[i] is 0 for absent components, never selected
        r.skip = true; r.done = true;
        if ((int)(mcu_row * m0) < g.trunc_bcv[0]) r.done = false;
        if (g.ncmp > 1 && (int)(mcu_row * m1) < g.trunc_bcv[1]) r.done = false;
    }
    if (i == 0) r.luma_y = r.curr_y;
    return r;
}

}  // namespace lepb200
