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
// Only the bins the grammar can reach are allocated (10 of 26 nz-count bins).
//
// Exponent chains are split.  Words k = 0..3 of a context take nearly all of its decisions on photographic input, so they
// form a 4-word HEAD (8 bytes; the 12 bit-length contexts of one position fill 3 whole 32-byte sectors: the heads start on
// a sector boundary and a position takes 96 bytes), and words k = 4..10 go to a
// TAIL region of 8-word rows in the same context order.  All heads are one array (DC, 7x7, edge), so the word after head
// word 3 is found from the address alone (m_exp_next).  The model starts with a FRONT region of small tables that nearly
// every block reads -- signs, DC residuals, the fixed top rows of the 7x7 count trees, the DC exponent heads --
// M_HOT words that the group decode kernel keeps in shared memory.
// ------------------------------------------------------------------------------------------------------
constexpr uint32_t M_SIGN = 0;                                       // [2][4][12]
constexpr uint32_t M_RESDC = M_SIGN + 2 * 4 * 12;                    // [12][10]
constexpr uint32_t M_NZ7T = M_RESDC + 12 * 10;                       // [2][10][8]: rows 3, 4, 5 of a 7x7 count tree (4 + 2 + 1 words, 1 pad)
constexpr uint32_t M_EXPH = M_NZ7T + 2 * 10 * 8 + 8;                 // exponent heads [context][4] (8 words of padding before them):
constexpr uint32_t M_EXPDC = M_EXPH;                                 //   [12][17]
constexpr uint32_t M_HOT = M_EXPDC + 12 * 17 * 4;                    // end of the front region
constexpr uint32_t M_EXP7 = M_HOT;                                   //   [2][10][49][12]
constexpr uint32_t M_EXPX = M_EXP7 + 2 * 10 * 49 * 12 * 4;           //   [2][8][15][12]
constexpr uint32_t M_EXPT = M_EXPX + 2 * 8 * 15 * 12 * 4;            // exponent tails [context][8]  (7 used)
constexpr uint32_t M_NZ7 = M_EXPT + 2 * (M_EXPT - M_EXPH);           // [2][10][56]: rows 0, 1, 2 of a 7x7 count tree (32 + 16 + 8 words)
constexpr uint32_t M_NZE = M_NZ7 + 2 * 10 * 56;                      // [2 kinds][2][8][8][3][4]  (kind 0 = 8x1 horizontal, 1 = 1x8 vertical)
constexpr uint32_t M_RESN = M_NZE + 2 * 2 * 8 * 8 * 3 * 4;           // [2][64][10][16]  (10 used)
constexpr uint32_t M_THR = M_RESN + 2 * 64 * 10 * 16;                // [2][256][8][128]
constexpr uint32_t M_TOTAL = M_THR + 2 * 256 * 8 * 128;              // u16 entries
static_assert(M_TOTAL < (1u << 20), "branch index must fit in 20 bits");
static_assert((M_TOTAL % 8) == 0 && (M_HOT % 8) == 0, "model zero fill uses 16-byte stores");
static_assert((M_EXPH % 16) == 0 && (M_HOT % 16) == 0 && (M_EXPX % 16) == 0 && (M_TOTAL % 16) == 0,
              "exponent heads start on a 32-byte sector in every model of a pool");
static_assert((M_NZ7T % 8) == 0 && (M_NZ7 % 8) == 0 && (M_NZE % 4) == 0, "count tree rows are read as 8- and 16-byte vectors");
constexpr size_t MODEL_BYTES = size_t(M_TOTAL) * 2;

// Interleaved model pool of the group decode kernel.  Segments of one batch hit largely the same contexts, but in a private
// model a 32-byte sector that one segment touches holds 15 words it never uses.  The group kernel therefore stores the models
// of MI_K consecutive jobs word pair by word pair: 4-byte unit u of model k of a block of W models sits at unit u * W + k,
// so the words that the W segments share fill whole sectors, and the segments one warp decodes in lock step (consecutive
// jobs) read the same sector when they are in the same state.  Every block holds W = MI_K models but the last one of a pool
// of n jobs, which holds the n % MI_K that are left: the pool is exactly n models long, as with private models.
// MI_K = 1 is the plain layout, one private model after the other.  Kernel A and the warp decode kernel keep private models.
#ifndef LEPB200_MODEL_INTERLEAVE
#define LEPB200_MODEL_INTERLEAVE 8
#endif
constexpr uint32_t MI_K = LEPB200_MODEL_INTERLEAVE;                  // models per interleave block
constexpr uint32_t MI_UNIT = 2;                                      // words per unit (4 bytes)
static_assert(MI_K >= 1 && (M_TOTAL % MI_UNIT) == 0, "a model is a whole number of units");
// models in the block of job j, in a pool of n jobs (j < n)
__host__ __device__ constexpr uint32_t mi_width(size_t j, size_t n) { return (uint32_t)(n - j / MI_K * MI_K < MI_K ? n - j / MI_K * MI_K : MI_K); }
// u16 offset of word `word` of model k (k < width) inside its block of `width` models; offset(w, k) = offset(w, 0) + offset(0, k)
__host__ __device__ constexpr uint32_t mi_offset(uint32_t word, uint32_t k, uint32_t width) {
    return ((word / MI_UNIT) * width + k) * MI_UNIT + word % MI_UNIT;
}
// u16 offset of job j's model (its word 0) in a pool of n jobs, which is n * M_TOTAL words long
__host__ __device__ constexpr size_t mi_model(size_t j, size_t n) {
    return j / MI_K * MI_K * M_TOTAL + mi_offset(0, (uint32_t)(j % MI_K), mi_width(j, n));
}
// For every width W, mi_offset(., ., W) is a bijection of [0, M_TOTAL) x [0, W) onto [0, W * M_TOTAL): it writes
// (word / MI_UNIT, k, word % MI_UNIT) in mixed radix (any, W, MI_UNIT).  Checked here on the first and last units of a block
// of every width (tests/test_emu_model_interleave.py checks whole blocks and whole pools on the host).
constexpr bool mi_round_trip(uint32_t width, uint32_t first, uint32_t n) {
    for (uint32_t off = first; off < first + n; ++off) {
        const uint32_t word = off / (MI_UNIT * width) * MI_UNIT + off % MI_UNIT, k = off / MI_UNIT % width;
        if (word >= M_TOTAL || mi_offset(word, k, width) != off) return false;
    }
    return true;
}
constexpr bool mi_bijection() {
    for (uint32_t w = 1; w <= MI_K; ++w)
        if (!mi_round_trip(w, 0, 4 * w * MI_UNIT) || !mi_round_trip(w, w * M_TOTAL - 4 * w * MI_UNIT, 4 * w * MI_UNIT) ||
            mi_offset(M_TOTAL - 1, w - 1, w) != w * M_TOTAL - 1)
            return false;
    return true;
}
static_assert(mi_bijection() && mi_model(MI_K, MI_K + 1) == (size_t)MI_K * M_TOTAL && mi_width(MI_K - 1, MI_K + 1) == MI_K &&
              mi_width(MI_K, MI_K + 1) == 1, "interleave is a bijection");

// 7x7 count tree: offset of row idx (2^(5-idx) words) in the tree's front part (idx >= 3) or rear part (idx < 3)
__host__ __device__ constexpr uint32_t nz7_row(int idx) { return idx >= 3 ? 8u - (16u >> (idx - 2)) : 64u - (64u >> idx); }
__host__ __device__ constexpr uint32_t m_nz7(int ci, int bin, int idx, int prefix) {
    return (idx >= 3 ? M_NZ7T + (uint32_t)(ci * 10 + bin) * 8u : M_NZ7 + (uint32_t)(ci * 10 + bin) * 56u) + nz7_row(idx) + (uint32_t)prefix;
}
__host__ __device__ constexpr uint32_t m_nze(int vertical, int ci, int eob, int nzb, int idx, int prefix) {
    return M_NZE + (((((vertical * 2 + ci) * 8 + eob) * 8 + nzb) * 3 + idx) << 2) + prefix;
}
// (a position-innermost variant of the three big tables was measured slower for both kernel A and the decode kernel, and dropped)
__host__ __device__ constexpr uint32_t m_resn(int ci, int coord, int bin) { return M_RESN + (((ci * 64 + coord) * 10 + bin) << 4); }
// exponent tables: the address of word k = 0 of a context (its head)
__host__ __device__ constexpr uint32_t m_exp7(int ci, int bin, int zz, int bsr) { return M_EXP7 + ((((ci * 10 + bin) * 49 + zz) * 12 + bsr) << 2); }
__host__ __device__ constexpr uint32_t m_expx(int ci, int ne, int zig15, int bsr) { return M_EXPX + ((((ci * 8 + ne) * 15 + zig15) * 12 + bsr) << 2); }
__host__ __device__ constexpr uint32_t m_expdc(int a, int b) { return M_EXPDC + ((a * 17 + b) << 2); }
// word k (0..10) of the exponent chain whose head is at `head`
__host__ __device__ constexpr uint32_t m_exp_word(uint32_t head, int k) { return k < 4 ? head + (uint32_t)k : M_EXPT + 2u * (head - M_EXPH) + (uint32_t)(k - 4); }
// word k + 1 of the chain, from the address of word k (k < 10)
__host__ __device__ constexpr uint32_t m_exp_next(uint32_t addr, int k) { return k == 3 ? M_EXPT + 2u * (addr - M_EXPH) - 6u : addr + 1u; }
__host__ __device__ constexpr uint32_t m_resdc(int lenmxm) { return M_RESDC + lenmxm * 10; }
__host__ __device__ constexpr uint32_t m_sign(int ci, int a, int b) { return M_SIGN + (ci * 4 + a) * 12 + b; }
__host__ __device__ constexpr uint32_t m_thr(int ci, int ctx, int len) { return M_THR + (((ci * 256 + ctx) * 8 + len) << 7); }

// no two tables overlap: the last word each index function can produce lies below the start of the next table
static_assert(m_sign(1, 3, 11) < M_RESDC && m_resdc(11) + 9 < M_NZ7T && m_nz7(1, 9, 5, 0) < M_EXPH, "front region tables overlap");
static_assert(m_exp_word(m_expdc(11, 16), 3) < M_EXP7 && m_exp_word(m_exp7(1, 9, 48, 11), 3) < M_EXPX &&
              m_exp_word(m_expx(1, 7, 14, 11), 3) < M_EXPT, "exponent heads overlap");
static_assert(m_exp_word(m_expdc(0, 0), 4) == M_EXPT && m_exp_next(m_exp_word(m_exp7(1, 2, 3, 4), 3), 3) == m_exp_word(m_exp7(1, 2, 3, 4), 4) &&
              m_exp_word(m_expx(1, 7, 14, 11), 10) < M_NZ7, "exponent tails overlap");
static_assert(m_nz7(1, 9, 0, 31) < M_NZE && m_nze(1, 1, 7, 7, 2, 3) < M_RESN && m_resn(1, 63, 9) + 15 < M_THR &&
              m_thr(1, 255, 7) + 127 < M_TOTAL, "model tables overlap");
// every row the group kernel reads unit by unit starts on a unit: rows 2, 1, 0 of each 7x7 count tree, rows 1, 0 of each edge tree
static_assert((m_nz7(0, 0, 0, 0) % MI_UNIT) == 0 && (m_nz7(0, 1, 0, 0) - m_nz7(0, 0, 0, 0)) % MI_UNIT == 0 &&
              nz7_row(1) % MI_UNIT == 0 && nz7_row(2) % MI_UNIT == 0 && (m_nze(0, 0, 0, 0, 0, 0) % MI_UNIT) == 0 &&
              (m_nze(0, 0, 0, 0, 1, 0) - m_nze(0, 0, 0, 0, 0, 0)) % MI_UNIT == 0 && (m_nze(0, 0, 0, 1, 0, 0) - m_nze(0, 0, 0, 0, 0, 0)) % MI_UNIT == 0,
              "count tree rows start on a unit in every model of an interleave block");

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
    int32_t coder;                   // decode: entropy coder of the image's streams (CODER_BOOL, CODER_ANS); a launch takes one coder's segments
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

// Entropy coders of a segment's stream: the VP8 bool coder of container versions 1, 2 and 4, or the two-state rANS coder of
// version 3 (the reference's -ans, ans_bool_reader.hh).  Same grammar and model layout; the rANS coder has its own update of
// the branch counts (branch_update_ans) and its own bits.
enum : int32_t { CODER_BOOL = 0, CODER_ANS = 1 };

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

// The rANS coder's model (ANSBoolReader::get and ANSBoolWriter::put call Branch::adv_record_obs_and_update, branch.hh:60-77):
// the observed count goes up, and from 255 it restarts at 129 while the other count is halved (rounded up); the probability
// is the same quotient with its low bit set, so it is never 0 and the special state of the bool coder's model never arises.
// Only a branch that was never updated (the zero word, counts (1, 1)) keeps its initial probability 128 (set_identity).
__device__ __forceinline__ uint32_t branch_prob_ans(uint32_t w, const uint32_t* __restrict__ s_rcp) {
    uint32_t lo = w & 0xff, hi = (w >> 8) & 0xff;
    uint32_t c0 = lo + 1, s = lo + hi + 2;
    return w == 0 ? 128u : __umulhi(c0 << 8, s_rcp[s]) | 1u;
}
__device__ __forceinline__ uint32_t branch_update_ans(uint32_t w, uint32_t obs) {
    uint32_t c0 = (w & 0xff) + 1, c1 = ((w >> 8) & 0xff) + 1;
    if (obs) { if (c1 == 255) { c1 = 129; c0 = (c0 + 1) >> 1; } else { c1 += 1; } }
    else { if (c0 == 255) { c0 = 129; c1 = (c1 + 1) >> 1; } else { c0 += 1; } }
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
