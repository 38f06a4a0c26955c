/*
 * lepton_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Scalar CPU restatement of dropbox/lepton's per-block context-modelled arithmetic coder
 * (the hot path named by BASELINE.json:north_star).  It exists so that the CUDA kernels in
 * lepton_b200/csrc can be checked bit-for-bit; nothing in the product links, imports or
 * executes it (only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may).
 *
 * Parity status: PINNED.  tests/test_oracle_golden.py checks this file against (a) the
 * per-segment arithmetic streams demuxed from .lep files written by the unmodified reference
 * binary (oracle/_ref/lepton, built by oracle/Makefile.ref) for the fixtures under
 * tests/golden/, with the coefficient planes taken from the reference's own `-ujg` dump, and
 * (b) the reference repo's golden .lep vectors (narrowrst.lep: test_suite/test_future_compat.sh).
 *
 * Each function cites the reference file:line it follows (paths relative to /root/reference).
 * Where the reference's scalar and SSE4 builds could diverge (16-bit wraparound) the SSE
 * semantics are followed, because the default `lepton` binary is the SSE4.2 build
 * (CMakeLists.txt:56,396).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ exit codes */
/* src/vp8/util/memory.hh:13-39 */
enum { LO_SUCCESS = 0, LO_ASSERTION_FAILURE = 1, LO_COEFFICIENT_OUT_OF_RANGE = 6, LO_STREAM_INCONSISTENT = 7,
       LO_UNSUPPORTED_JPEG_WITH_ZERO_IDCT_0 = 43, LO_OUTPUT_OVERFLOW = 100 };

/* ------------------------------------------------------------------ static tables */
/* src/vp8/model/jpeg_meta.hh:13-23 (zigzag: raster index -> zigzag position) */
static const uint8_t k_zigzag[64] = {
    0, 1, 5, 6, 14, 15, 27, 28, 2, 4, 7, 13, 16, 26, 29, 42, 3, 8, 12, 17, 25, 30, 41, 43, 9, 11, 18, 24, 31, 40, 44, 53,
    10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};
/* src/vp8/util/aligned_block.hh:32-44 (aligned index -> raster index) */
static const uint8_t k_aligned_to_raster[64] = {
    9, 10, 17, 25, 18, 11, 12, 19, 26, 33, 41, 34, 27, 20, 13, 14, 21, 28, 35, 42, 49, 57, 50, 43, 36,
    29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63,
    0, 1, 2, 3, 4, 5, 6, 7, 8, 16, 24, 32, 40, 48, 56};
static uint8_t k_raster_to_aligned[64]; /* inverse, built in lo_init_tables (aligned_block.hh:46-55) */
/* src/vp8/model/jpeg_meta.hh:72-170, row NUM_NONZEROS_BINS-1 == 9 (model.hh:562-564) */
static const uint8_t k_nonzero_to_bin[50] = {
    0, 1, 2, 3, 4, 4, 5, 5, 5, 6, 6, 6, 6, 7, 7, 7, 7, 7, 7, 7, 7, 8, 8, 8, 8,
    8, 8, 8, 8, 8, 8, 8, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9};
/* src/vp8/model/jpeg_meta.hh:48-58 */
static const int k_icos_base_8192_scaled[64] = {
    8192, 8192, 8192, 8192, 8192, 8192, 8192, 8192, 11363, 9633, 6436, 2260, -2260, -6436, -9633, -11363,
    10703, 4433, -4433, -10703, -10703, -4433, 4433, 10703, 9633, -2260, -11363, -6436, 6436, 11363, 2260, -9633,
    8192, -8192, -8192, 8192, 8192, -8192, -8192, 8192, 6436, -11363, 2260, 9633, -9633, -2260, 11363, -6436,
    4433, -10703, 10703, -4433, -4433, 10703, -10703, 4433, 2260, -6436, 9633, -11363, 11363, -9633, 6436, -2260};
/* src/vp8/model/model.hh:264-274 */
static const uint16_t k_freqmax[64] = {
    1024, 931, 985, 968, 1020, 968, 1020, 1020, 932, 858, 884, 840, 932, 838, 854, 854,
    985, 884, 871, 875, 985, 878, 871, 854, 967, 841, 876, 844, 967, 886, 870, 837,
    1020, 932, 985, 967, 1020, 969, 1020, 1020, 969, 838, 878, 886, 969, 838, 969, 838,
    1020, 854, 871, 870, 1010, 969, 1020, 1020, 1020, 854, 854, 838, 1020, 838, 1020, 838};

static int g_tables_ready = 0;
static void lo_init_tables(void) {
    if (g_tables_ready) return;
    for (int a = 0; a < 64; ++a) k_raster_to_aligned[k_aligned_to_raster[a]] = (uint8_t)a;
    g_tables_ready = 1;
}

/* src/vp8/model/numeric.hh:394-403 */
static inline int bit_length(uint32_t v) { return v ? 32 - __builtin_clz(v) : 0; }
static inline int iabs(int v) { return v < 0 ? -v : v; }
static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

/* ------------------------------------------------------------------ Branch + Model */
/* src/vp8/model/branch.hh:11-128 */
typedef struct { uint8_t c0, c1, p; } Branch;

/* record_obs_and_update, branch.hh:82-100.  optimize() (branch.hh:108-120) is exact floor division
 * (fast_divide18bit_by_10bit == num/denom, test_suite/test_invariants.cc:500-531). */
static inline void branch_update(Branch *b, int obs) {
    unsigned f = b->c0, t = b->c1;
    uint8_t *c = obs ? &b->c1 : &b->c0;
    int overflow = ((*c)++ == 0xff);
    if (overflow) {
        int neverseen = (obs ? b->c0 : b->c1) == 1;
        if (neverseen) {
            *c = 0xff;
            b->p = obs ? 0 : 255;
        } else {
            b->c0 = (uint8_t)((1 + f) >> 1);
            b->c1 = (uint8_t)((1 + t) >> 1);
            *c = 129;
            b->p = (uint8_t)(((unsigned)b->c0 << 8) / ((unsigned)b->c0 + b->c1));
        }
    } else {
        b->p = (uint8_t)(((unsigned)b->c0 << 8) / (f + t + 1));
    }
}

/* src/vp8/model/model.hh:60-127 (array shapes) */
typedef struct {
    Branch nz7x7[2][26][6][32];
    Branch nz1x8[2][8][8][3][4];
    Branch nz8x1[2][8][8][3][4];
    Branch res_noise[2][64][10][10];
    Branch res_noise_dc[12][10];
    Branch res_thresh[2][256][8][128];
    Branch exp7x7[2][10][49][12][11];
    Branch exp_x[2][10][15][12][11];
    Branch exp_dc[12][17][11];
    Branch sign[2][4][12];
} Model;

static void model_reset(Model *m) { /* model.hh:114-125, branch.hh:31-35 */
    Branch *b = (Branch *)m;
    size_t n = sizeof(Model) / sizeof(Branch);
    for (size_t i = 0; i < n; ++i) { b[i].c0 = 1; b[i].c1 = 1; b[i].p = 128; }
}

/* ------------------------------------------------------------------ bool coder */
/* src/vp8/encoder/boolwriter.hh:48-118, boolwriter.cc:17-35 */
typedef struct {
    uint32_t low, range; int count; size_t pos; uint8_t *buf; size_t cap; int overflow;
} BoolWriter;

/* bool-coder regime counters (lo_bool_counts): bytes a carry changes (the 0xff bytes it turns into zeros, plus the byte it
 * increments) -- the longest such walk and the number of walks of 64 bytes or more -- and the streams that end with the
 * extra zero byte of vpx_stop_encode */
static uint64_t g_bw_walk_max, g_bw_walk_long, g_bw_stop_zero;

static void bw_write(BoolWriter *w, int bit, int prob) {
    uint32_t split = 1 + (((w->range - 1) * (uint32_t)prob) >> 8);
    uint32_t range = split, low = w->low;
    int count = w->count;
    if (bit) { low += split; range = w->range - split; }
    int shift = __builtin_clz(range) - 24; /* == vpx_norm[range] for 1 <= range <= 255 */
    range <<= shift;
    count += shift;
    if (count >= 0) {
        int offset = shift - count;
        if ((low << (offset - 1)) & 0x80000000u) {
            long x = (long)w->pos - 1;
            while (x >= 0 && w->buf[x] == 0xff) { w->buf[x] = 0; x--; }
            w->buf[x] += 1;
            const uint64_t walk = (uint64_t)((long)w->pos - x);
            if (walk > g_bw_walk_max) g_bw_walk_max = walk;
            if (walk >= 64) ++g_bw_walk_long;
        }
        if (w->pos + 2 >= w->cap) { w->overflow = 1; w->pos = 0; }
        w->buf[w->pos++] = (uint8_t)(low >> (24 - offset));
        low <<= offset;
        shift = count;
        low &= 0xffffff;
        count -= 8;
    }
    low <<= shift;
    w->count = count; w->low = low; w->range = range;
}
static void bw_start(BoolWriter *w, uint8_t *buf, size_t cap) {
    w->low = 0; w->range = 255; w->count = -24; w->buf = buf; w->pos = 0; w->cap = cap; w->overflow = 0;
    bw_write(w, 0, 128);
}
static void bw_stop(BoolWriter *w) {
    for (int i = 0; i < 32; i++) bw_write(w, 0, 128);
    if ((w->buf[w->pos - 1] & 0xe0) == 0xc0) { w->buf[w->pos++] = 0; ++g_bw_stop_zero; }
}

/* src/vp8/decoder/boolreader.hh:184-258,376-416, boolreader.cc:26-35.  The reference refills a 64-bit
 * big-endian window from a packet rope and supplies zero bits past the end of the stream; the decoded
 * bit sequence depends only on the byte stream, so the window is refilled a byte at a time here. */
typedef struct { uint64_t value; uint32_t range; int count; const uint8_t *p, *end; } BoolReader;

static void br_fill(BoolReader *r) {
    int shift = 64 - 8 - (r->count + 8);
    while (shift >= 0) {
        uint64_t byte = (r->p < r->end) ? *r->p++ : 0;
        r->value |= byte << shift;
        r->count += 8;
        shift -= 8;
    }
}
static int br_read(BoolReader *r, int prob) {
    uint32_t split = (r->range * (uint32_t)prob + (256 - (uint32_t)prob)) >> 8;
    if (r->count < 0) br_fill(r);
    uint64_t bigsplit = (uint64_t)split << 56;
    int bit = r->value >= bigsplit;
    uint32_t range;
    if (bit) { range = r->range - split; r->value -= bigsplit; } else { range = split; }
    int shift = __builtin_clz(range) - 24;
    r->range = range << shift;
    r->value <<= shift;
    r->count -= shift;
    return bit;
}
static void br_init(BoolReader *r, const uint8_t *p, size_t n) {
    r->value = 0; r->count = -8; r->range = 255; r->p = p; r->end = p + n;
    br_fill(r);
    (void)br_read(r, 128); /* marker bit */
}

/* ------------------------------------------------------------------ geometry / per-image tables */
typedef struct {
    int32_t ncmp;
    int32_t bch[3], bcv[3];      /* componentInfo.bch / .bcv (block_based_image.hh width_, original_height()) */
    int32_t trunc_bcv[3];        /* UncompressedComponents::get_max_coded_heights (uncompressed_components.hh:69-76) */
    int32_t trunc_bc[3];         /* component_size_in_blocks (uncompressed_components.hh:241-243) */
    int32_t mcuv;                /* get_mcu_count_vertical */
    uint16_t q_zigzag[3][64];    /* get_quantization_tables(cmp): DQT in zigzag order */
} lo_geometry;

typedef struct {
    uint16_t q[64];        /* raster order, model.hh:248-250 */
    int32_t icos_x[64];    /* icos_idct_edge_8192_dequantized_x, model.hh:254 */
    int32_t icos_y[64];    /* icos_idct_edge_8192_dequantized_y, model.hh:255 */
    uint8_t min_noise_threshold[64]; /* model.hh:277-289 */
} QuantTables;

static int quant_tables_init(QuantTables *t, const uint16_t zz[64]) {
    for (int i = 0; i < 64; ++i) t->q[i] = zz[k_zigzag[i]];
    for (int r = 0; r < 8; ++r) {
        for (int i = 0; i < 8; ++i) {
            t->icos_x[r * 8 + i] = k_icos_base_8192_scaled[i * 8] * t->q[i * 8 + r];
            t->icos_y[r * 8 + i] = k_icos_base_8192_scaled[i * 8] * t->q[r * 8 + i];
        }
        if (t->icos_x[r * 8] == 0 || t->icos_y[r * 8] == 0) return LO_UNSUPPORTED_JPEG_WITH_ZERO_IDCT_0; /* model.hh:257-262 */
    }
    for (int c = 0; c < 64; ++c) {
        uint16_t fm = (uint16_t)(k_freqmax[c] + t->q[c] - 1);
        if (t->q[c]) fm /= t->q[c];
        int len = bit_length(fm);
        t->min_noise_threshold[c] = (uint8_t)(len > 7 ? len - 7 : 0);
    }
    return 0;
}

/* src/vp8/util/block_context.hh:17-95 */
typedef struct { int16_t edge[16]; uint8_t nz; } NeighborSummary;

typedef struct {
    const lo_geometry *g;
    QuantTables qt[3];
    Model *model;
    NeighborSummary *ns[3];      /* 2 * bch entries each: ring rows (y & 1), block_based_image.hh:97-100 */
    int16_t *planes[3];
    int encode;
    BoolWriter bw;
    BoolReader br;
    uint64_t ndecisions;
    int err;
} Codec;

static inline int code_bit(Codec *c, Branch *b, int bit) {
    /* vpx_bool_writer.hh:43-60 / vpx_bool_reader.hh:45-57 */
    if (c->encode) bw_write(&c->bw, bit, b->p);
    else bit = br_read(&c->br, b->p);
    branch_update(b, bit);
    c->ndecisions++;
    return bit;
}

/* ------------------------------------------------------------------ regime counters
 * Each site below is a place where the reference's arithmetic wraps, truncates or caps.  Beside the wrapped value the
 * oracle computes the exact one (int64, no cap); when they differ the site's counter goes up.  The counters change
 * nothing that is coded: they show which of these regimes a test input really reaches.  (The cap of 16 on the bit length
 * of the DC offset uncertainty has no site: the estimates are int16, so |unc2| <= 32768 and its bit length never
 * exceeds 16.) */
enum {
    RG_IDCT_INT32_WRAP,      /* an IDCT output whose int32 computation wrapped */
    RG_IDCT_INT16_PIXEL,     /* an IDCT output pixel that does not fit the int16 it is stored in */
    RG_DC_EST_INT16,         /* a DC estimate from a neighbour edge pixel that wrapped in int16 */
    RG_EDGE_INT16,           /* an edge pixel of the neighbour summary that wrapped in int16 */
    RG_QDC_INT16,            /* q0 * dc wrapped in int16 */
    RG_LAK_UINT32_WRAP,      /* the Lakhani predictor's sum wrapped in 32 bits */
    RG_SIGN_CTX_INT16,       /* (int16_t)prior of the edge sign context differs from prior */
    RG_THR_CTX_MASK,         /* |prior| > 0xffff: the threshold context keeps only its low 16 bits */
    RG_THR_CTX_CAP255,       /* the threshold context (|prior| & 0xffff) >> min_thr capped at 255 */
    RG_BSR_CAP1023,          /* |prior| capped at 1023 for the exponent context */
    RG_LEN_MXM_CAP11,        /* DC uncertainty bit length capped at 11 */
    RG_THR_SO_SAT127,        /* the threshold bits' context index saturated at 127 */
    RG_ADV_WRAP_POS,         /* adv_unpredict wrapped a value above +1024 */
    RG_ADV_WRAP_NEG,         /* adv_unpredict wrapped a value below -1024 */
    RG_AC_LEN11,             /* an AC coefficient of the largest codable length, 11 */
    RG_REFUSE_DC,            /* status 6: a DC that adv_unpredict cannot round-trip */
    RG_REFUSE_DC_LEN,        /* status 6: a DC residual that round-trips but is longer than 11 bits */
    RG_REFUSE_AC,            /* status 6: a coefficient longer than 11 bits */
    RG_COUNT
};
static const char *const k_regime_names[RG_COUNT] = {
    "idct_int32_wrap", "idct_int16_pixel", "dc_est_int16", "edge_int16", "qdc_int16", "lak_uint32_wrap",
    "sign_ctx_int16", "thr_ctx_mask", "thr_ctx_cap255", "bsr_cap1023", "len_mxm_cap11",
    "thr_so_sat127", "adv_wrap_pos", "adv_wrap_neg", "ac_len11", "refuse_dc", "refuse_dc_len", "refuse_ac"};
static uint64_t g_regime[RG_COUNT];
#define REGIME(site, cond) do { if (cond) ++g_regime[site]; } while (0)

/* ------------------------------------------------------------------ IDCT (src/lepton/idct.cc:36-161; SSE form :196-355) */
/* the same IDCT in exact int64 arithmetic (nothing wraps): what idct_sans_dc would give without its int32 wrap */
static void idct_exact(const int16_t *blk /*aligned*/, const uint16_t q[64], int64_t out[64]) {
    const int64_t w1 = 2841, w2 = 2676, w3 = 2408, w5 = 1609, w6 = 1108, w7 = 565, r2 = 181;
    int64_t im[64];
    for (int y = 0; y < 8; ++y) {
        int64_t c[8];
        for (int i = 0; i < 8; ++i) c[i] = (y == 0 && i == 0) ? 0 : (int64_t)blk[k_raster_to_aligned[y * 8 + i]] * q[y * 8 + i];
        int64_t x0 = c[0] * 2048 + 128, x1 = c[4] * 2048, x2 = c[6], x3 = c[2], x4 = c[1], x5 = c[7], x6 = c[5], x7 = c[3];
        int64_t x8 = w7 * (x4 + x5);
        x4 = x8 + (w1 - w7) * x4; x5 = x8 - (w1 + w7) * x5;
        x8 = w3 * (x6 + x7);
        x6 = x8 - (w3 - w5) * x6; x7 = x8 - (w3 + w5) * x7;
        x8 = x0 + x1; x0 -= x1;
        x1 = w6 * (x3 + x2);
        x2 = x1 - (w2 + w6) * x2; x3 = x1 + (w2 - w6) * x3;
        x1 = x4 + x6; x4 -= x6; x6 = x5 + x7; x5 -= x7;
        x7 = x8 + x3; x8 -= x3; x3 = x0 + x2; x0 -= x2;
        x2 = (r2 * (x4 + x5) + 128) >> 8; x4 = (r2 * (x4 - x5) + 128) >> 8;
        int64_t *o = im + y * 8;
        o[0] = (x7 + x1) >> 8; o[1] = (x3 + x2) >> 8; o[2] = (x0 + x4) >> 8; o[3] = (x8 + x6) >> 8;
        o[4] = (x8 - x6) >> 8; o[5] = (x0 - x4) >> 8; o[6] = (x3 - x2) >> 8; o[7] = (x7 - x1) >> 8;
    }
    for (int x = 0; x < 8; ++x) {
        int64_t y0 = im[x] * 256 + 8192, y1 = im[32 + x] * 256;
        int64_t y2 = im[48 + x], y3 = im[16 + x], y4 = im[8 + x], y5 = im[56 + x], y6 = im[40 + x], y7 = im[24 + x];
        int64_t y8 = w7 * (y4 + y5) + 4;
        y4 = (y8 + (w1 - w7) * y4) >> 3; y5 = (y8 - (w1 + w7) * y5) >> 3;
        y8 = w3 * (y6 + y7) + 4;
        y6 = (y8 - (w3 - w5) * y6) >> 3; y7 = (y8 - (w3 + w5) * y7) >> 3;
        y8 = y0 + y1; y0 -= y1;
        y1 = w6 * (y3 + y2) + 4;
        y2 = (y1 - (w2 + w6) * y2) >> 3; y3 = (y1 + (w2 - w6) * y3) >> 3;
        y1 = y4 + y6; y4 -= y6; y6 = y5 + y7; y5 -= y7;
        y7 = y8 + y3; y8 -= y3; y3 = y0 + y2; y0 -= y2;
        y2 = (r2 * (y4 + y5) + 128) >> 8; y4 = (r2 * (y4 - y5) + 128) >> 8;
        out[x] = (y7 + y1) >> 11; out[8 + x] = (y3 + y2) >> 11; out[16 + x] = (y0 + y4) >> 11; out[24 + x] = (y8 + y6) >> 11;
        out[32 + x] = (y8 - y6) >> 11; out[40 + x] = (y0 - y4) >> 11; out[48 + x] = (y3 - y2) >> 11; out[56 + x] = (y7 - y1) >> 11;
    }
}

static void idct_sans_dc(const int16_t *blk /*aligned*/, const uint16_t q[64], int16_t outp[64]) {
    enum { w1 = 2841, w2 = 2676, w3 = 2408, w5 = 1609, w6 = 1108, w7 = 565, r2 = 181,
           w1pw7 = w1 + w7, w1mw7 = w1 - w7, w2pw6 = w2 + w6, w2mw6 = w2 - w6, w3pw5 = w3 + w5, w3mw5 = w3 - w5 };
    int32_t im[64], wide[64];
#define CR(i) ((int32_t)blk[k_raster_to_aligned[i]])
#define U(x) ((uint32_t)(x))
    for (int y = 0; y < 8; ++y) {
        int y8 = y * 8;
        int32_t x0 = (int32_t)(U(y == 0 ? 0 : (int32_t)(U(CR(y8) * q[y8]) << 11)) + 128u);
        int32_t x1 = (int32_t)(U(CR(y8 + 4) * q[y8 + 4]) << 11);
        int32_t x2 = CR(y8 + 6) * q[y8 + 6];
        int32_t x3 = CR(y8 + 2) * q[y8 + 2];
        int32_t x4 = CR(y8 + 1) * q[y8 + 1];
        int32_t x5 = CR(y8 + 7) * q[y8 + 7];
        int32_t x6 = CR(y8 + 5) * q[y8 + 5];
        int32_t x7 = CR(y8 + 3) * q[y8 + 3];
        int32_t x8 = (int32_t)(U(w7) * U(x4 + x5));
        x4 = (int32_t)(U(x8) + U(w1mw7) * U(x4));
        x5 = (int32_t)(U(x8) - U(w1pw7) * U(x5));
        x8 = (int32_t)(U(w3) * U(x6 + x7));
        x6 = (int32_t)(U(x8) - U(w3mw5) * U(x6));
        x7 = (int32_t)(U(x8) - U(w3pw5) * U(x7));
        x8 = (int32_t)(U(x0) + U(x1));
        x0 = (int32_t)(U(x0) - U(x1));
        x1 = (int32_t)(U(w6) * U(x3 + x2));
        x2 = (int32_t)(U(x1) - U(w2pw6) * U(x2));
        x3 = (int32_t)(U(x1) + U(w2mw6) * U(x3));
        x1 = (int32_t)(U(x4) + U(x6));
        x4 = (int32_t)(U(x4) - U(x6));
        x6 = (int32_t)(U(x5) + U(x7));
        x5 = (int32_t)(U(x5) - U(x7));
        x7 = (int32_t)(U(x8) + U(x3));
        x8 = (int32_t)(U(x8) - U(x3));
        x3 = (int32_t)(U(x0) + U(x2));
        x0 = (int32_t)(U(x0) - U(x2));
        x2 = (int32_t)(U(r2) * U(x4 + x5) + 128u) >> 8;
        x4 = (int32_t)(U(r2) * U(x4 - x5) + 128u) >> 8;
        im[y8 + 0] = (int32_t)(U(x7) + U(x1)) >> 8;
        im[y8 + 1] = (int32_t)(U(x3) + U(x2)) >> 8;
        im[y8 + 2] = (int32_t)(U(x0) + U(x4)) >> 8;
        im[y8 + 3] = (int32_t)(U(x8) + U(x6)) >> 8;
        im[y8 + 4] = (int32_t)(U(x8) - U(x6)) >> 8;
        im[y8 + 5] = (int32_t)(U(x0) - U(x4)) >> 8;
        im[y8 + 6] = (int32_t)(U(x3) - U(x2)) >> 8;
        im[y8 + 7] = (int32_t)(U(x7) - U(x1)) >> 8;
    }
    for (int x = 0; x < 8; ++x) {
        int32_t y0 = (int32_t)((U(im[x]) << 8) + 8192u);
        int32_t y1 = (int32_t)(U(im[32 + x]) << 8);
        int32_t y2 = im[48 + x], y3 = im[16 + x], y4 = im[8 + x], y5 = im[56 + x], y6 = im[40 + x], y7 = im[24 + x];
        int32_t y8 = (int32_t)(U(w7) * U(y4 + y5) + 4u);
        y4 = (int32_t)(U(y8) + U(w1mw7) * U(y4)) >> 3;
        y5 = (int32_t)(U(y8) - U(w1pw7) * U(y5)) >> 3;
        y8 = (int32_t)(U(w3) * U(y6 + y7) + 4u);
        y6 = (int32_t)(U(y8) - U(w3mw5) * U(y6)) >> 3;
        y7 = (int32_t)(U(y8) - U(w3pw5) * U(y7)) >> 3;
        y8 = (int32_t)(U(y0) + U(y1));
        y0 = (int32_t)(U(y0) - U(y1));
        y1 = (int32_t)(U(w6) * U(y3 + y2) + 4u);
        y2 = (int32_t)(U(y1) - U(w2pw6) * U(y2)) >> 3;
        y3 = (int32_t)(U(y1) + U(w2mw6) * U(y3)) >> 3;
        y1 = (int32_t)(U(y4) + U(y6));
        y4 = (int32_t)(U(y4) - U(y6));
        y6 = (int32_t)(U(y5) + U(y7));
        y5 = (int32_t)(U(y5) - U(y7));
        y7 = (int32_t)(U(y8) + U(y3));
        y8 = (int32_t)(U(y8) - U(y3));
        y3 = (int32_t)(U(y0) + U(y2));
        y0 = (int32_t)(U(y0) - U(y2));
        y2 = (int32_t)(U(r2) * U(y4 + y5) + 128u) >> 8;
        y4 = (int32_t)(U(r2) * U(y4 - y5) + 128u) >> 8;
        wide[x] = ((int32_t)(U(y7) + U(y1)) >> 11);
        wide[8 + x] = ((int32_t)(U(y3) + U(y2)) >> 11);
        wide[16 + x] = ((int32_t)(U(y0) + U(y4)) >> 11);
        wide[24 + x] = ((int32_t)(U(y8) + U(y6)) >> 11);
        wide[32 + x] = ((int32_t)(U(y8) - U(y6)) >> 11);
        wide[40 + x] = ((int32_t)(U(y0) - U(y4)) >> 11);
        wide[48 + x] = ((int32_t)(U(y3) - U(y2)) >> 11);
        wide[56 + x] = ((int32_t)(U(y7) - U(y1)) >> 11);
    }
    int64_t exact[64];
    idct_exact(blk, q, exact);
    for (int i = 0; i < 64; ++i) {
        outp[i] = (int16_t)wide[i];
        REGIME(RG_IDCT_INT32_WRAP, wide[i] != exact[i]);
        REGIME(RG_IDCT_INT16_PIXEL, outp[i] != wide[i]);
    }
#undef CR
#undef U
}

/* ------------------------------------------------------------------ predictors */
typedef struct {
    const int16_t *here, *left, *above, *above_left; /* aligned-order blocks; NULL when not present */
    NeighborSummary *ns_here, *ns_left, *ns_above;
} BlockCtx;

/* compute_aavrg_vec, model.hh:895-924 (16-bit lanes) */
static inline int16_t aavrg(const BlockCtx *b, int aligned_zz) {
    if (!b->left && !b->above) return 0;
    uint16_t l = b->left ? (uint16_t)iabs(b->left[aligned_zz]) : 0;
    if (b->left && !b->above) return (int16_t)l;
    uint16_t a = (uint16_t)iabs(b->above[aligned_zz]);
    if (!b->left) return (int16_t)a;
    uint16_t total = (uint16_t)(l + a);
    total = (uint16_t)(total * 13);
    total = (uint16_t)(total + (uint16_t)((uint16_t)iabs(b->above_left[aligned_zz]) * 6));
    return (int16_t)(total >> 5);
}

/* compute_lak, model.hh:1033-1071 (== compute_lak_vec :928-958 in wrapping int32) */
static int32_t lak(const BlockCtx *b, const QuantTables *qt, int band) {
    int32_t cx[8], ca[8];
    const int32_t *icos;
    if ((band & 7) && b->above) {
        for (int i = 0; i < 8; ++i) {
            int cur = band + i * 8;
            cx[i] = i ? b->here[k_raster_to_aligned[cur]] : 0;
            ca[i] = b->above[k_raster_to_aligned[cur]];
        }
        icos = qt->icos_x + band * 8;
    } else if ((band & 7) == 0 && b->left) {
        for (int i = 0; i < 8; ++i) {
            int cur = band + i;
            cx[i] = i ? b->here[k_raster_to_aligned[cur]] : 0;
            ca[i] = b->left[k_raster_to_aligned[cur]];
        }
        icos = qt->icos_y + band;
    } else {
        return 0;
    }
    uint32_t pred = (uint32_t)ca[0] * (uint32_t)icos[0];
    int64_t exact = (int64_t)ca[0] * icos[0];
    for (int i = 1; i < 8; ++i) {
        int sign = (i & 1) ? 1 : -1;
        pred -= (uint32_t)icos[i] * (uint32_t)(cx[i] + sign * ca[i]);
        exact -= (int64_t)icos[i] * (cx[i] + sign * ca[i]);
    }
    REGIME(RG_LAK_UINT32_WRAP, (int32_t)pred != exact);
    return (int32_t)pred / icos[0];
}

/* shift_right_round_zero_epi16(v, 1): model.hh:673 -- int16 truncating halving */
static inline int16_t half_rz16(int16_t d) { return (int16_t)(d / 2); }

/* adv_predict_dc_pix, model.hh:674-784 (SSE branch :682-729) */
static int adv_predict_dc_pix(const BlockCtx *b, const QuantTables *qt, int16_t pix[64], int *unc, int *unc2) {
    idct_sans_dc(b->here, qt->q, pix);
    int16_t est[16];
    memset(est, 0, sizeof(est));
    int32_t avgmed = 0;
    *unc = 0; *unc2 = 0;
    int has_left = b->left != NULL, has_above = b->above != NULL;
    if (has_left || has_above) {
        if (has_above) {
            int16_t *dst = est + (has_left ? 8 : 0);
            for (int i = 0; i < 8; ++i) {
                int16_t delta = (int16_t)(pix[i] - pix[i + 8]);
                int16_t recentered = (int16_t)(pix[i] + 1024);
                dst[i] = (int16_t)((int16_t)(b->ns_above->edge[8 + i] - half_rz16(delta)) - recentered);
                REGIME(RG_DC_EST_INT16, dst[i] != b->ns_above->edge[8 + i] - (pix[i] - pix[i + 8]) / 2 - (pix[i] + 1024));
            }
        }
        if (has_left) {
            for (int i = 0; i < 8; ++i) {
                int16_t delta = (int16_t)(pix[i * 8] - pix[i * 8 + 1]);
                int16_t recentered = (int16_t)(pix[i * 8] + 1024);
                est[i] = (int16_t)((int16_t)(b->ns_left->edge[i] - half_rz16(delta)) - recentered);
                REGIME(RG_DC_EST_INT16, est[i] != b->ns_left->edge[i] - (pix[i * 8] - pix[i * 8 + 1]) / 2 - (pix[i * 8] + 1024));
            }
        }
        int32_t avg_h_v[2] = {0, 0};
        int32_t min_dc = est[0], max_dc = est[0];
        int which = 0;
        for (int vert = 0; vert != 2; ++vert) {
            for (int i = 0; i < 8; ++which, ++i) {
                int16_t cur = est[which];
                avg_h_v[vert] += cur;
                if (min_dc > cur) min_dc = cur;
                if (max_dc < cur) max_dc = cur;
            }
            if (!has_above || !has_left) { avg_h_v[1] = avg_h_v[0]; break; }
        }
        int32_t overall = (avg_h_v[0] + avg_h_v[1]) >> 1;
        avgmed = overall;
        *unc = (max_dc - min_dc) >> 3;
        avg_h_v[0] -= avgmed;
        avg_h_v[1] -= avgmed;
        int32_t far_afield = avg_h_v[1];
        if (iabs(avg_h_v[0]) < iabs(avg_h_v[1])) far_afield = avg_h_v[0];
        *unc2 = far_afield >> 3;
    }
    return ((avgmed / (int)qt->q[0] + 4) >> 3);
}

/* adv_predict_or_unpredict_dc, model.hh:823-832 */
static inline int adv_unpredict(int16_t saved_dc, int recover, int pred) {
    int max_value = 1 << 10, min_value = -max_value, adj = 2 * max_value + 1;
    int r = saved_dc + (recover ? pred : -pred);
    REGIME(RG_ADV_WRAP_NEG, r < min_value);
    REGIME(RG_ADV_WRAP_POS, r > max_value);
    if (r < min_value) r += adj;
    if (r > max_value) r -= adj;
    return r;
}

/* NeighborSummary::set_horizontal / set_vertical, block_context.hh:44-78 (SSE: 16-bit lanes) */
static void ns_set_edges(NeighborSummary *ns, const int16_t pix[64], const uint16_t q[64], int16_t dc) {
    int16_t qdc = (int16_t)((uint16_t)q[0] * (uint16_t)dc);
    const int64_t qdc_exact = (int64_t)q[0] * dc;
    REGIME(RG_QDC_INT16, qdc != qdc_exact);
    for (int i = 0; i < 8; ++i) {
        int16_t delta = (int16_t)(pix[56 + i] - pix[48 + i]);
        ns->edge[8 + i] = (int16_t)(pix[56 + i] + half_rz16(delta) + 1024 + qdc);
        REGIME(RG_EDGE_INT16, ns->edge[8 + i] != pix[56 + i] + (pix[56 + i] - pix[48 + i]) / 2 + 1024 + qdc_exact);
        int16_t deltav = (int16_t)(pix[i * 8 + 7] - pix[i * 8 + 6]);
        ns->edge[i] = (int16_t)(pix[i * 8 + 7] + half_rz16(deltav) + 1024 + qdc);
        REGIME(RG_EDGE_INT16, ns->edge[i] != pix[i * 8 + 7] + (pix[i * 8 + 7] - pix[i * 8 + 6]) / 2 + 1024 + qdc_exact);
    }
}

/* ------------------------------------------------------------------ per-block token grammar */
/* nonzero_counts_7x7, model.hh:463-485 */
static Branch *nz7x7_slice(Codec *c, int ci, const BlockCtx *b) {
    int above = b->above ? b->ns_above->nz : 0, left = b->left ? b->ns_left->nz : 0;
    int ctx = 0;
    if (b->above && !b->left) ctx = (above + 1) / 2;
    else if (b->left && !b->above) ctx = (left + 1) / 2;
    else if (b->left && b->above) ctx = (above + left + 2) / 4;
    return &c->model->nz7x7[ci][k_nonzero_to_bin[ctx]][0][0];
}

/* code one magnitude/sign/residual: shared shape of encoder.cc:256-283 / decoder.cc:212-240 */

/* encode_one_edge (encoder.cc:39-164) / decode_one_edge (decoder.cc:27-141) */
static void code_one_edge(Codec *c, int cmp, int ci, const BlockCtx *b, int16_t *here_mut, int horizontal,
                          int nz7x7, int est_eob) {
    const QuantTables *qt = &c->qt[cmp];
    Branch(*eob)[4] = horizontal ? c->model->nz8x1[ci][est_eob][(nz7x7 + 3) / 7] : c->model->nz1x8[ci][est_eob][(nz7x7 + 3) / 7];
    int delta = horizontal ? 1 : 8, zig15 = horizontal ? 0 : 7;
    int aligned_off = horizontal ? 50 : 57; /* raster_to_aligned(1) / (8); consecutive (aligned_block.hh:43-44) */
    int ne = 0;
    if (c->encode)
        for (int k = 1; k < 8; ++k) ne += b->here[k_raster_to_aligned[k * delta]] != 0;
    int so_far = 0;
    int ne_dec = 0;
    for (int i = 2; i >= 0; --i) {
        int bit = code_bit(c, &eob[i][so_far], (ne >> i) & 1);
        ne_dec |= bit << i;
        so_far = (so_far << 1) | bit;
    }
    if (!c->encode) ne = ne_dec;
    if (ne > 7) { c->err = LO_STREAM_INCONSISTENT; return; }
    int coord = delta;
    for (int lane = 0; lane < 7 && ne; ++lane, coord += delta, ++zig15) {
        int32_t prior = lak(b, qt, coord);
        int nzbin = ne;
        int bsr = bit_length((uint32_t)imin(iabs(prior), 1023));
        REGIME(RG_BSR_CAP1023, iabs(prior) > 1023);
        Branch *exp = c->model->exp_x[ci][nzbin][zig15][bsr];
        int16_t coef = c->encode ? b->here[aligned_off + lane] : 0;
        uint16_t abs_coef = (uint16_t)iabs(coef);
        int length = bit_length(abs_coef);
        int dec_len = 0, nonzero = 0;
        for (int i = 0; i < 11; ++i) {
            int bit = code_bit(c, &exp[i], length != i);
            if (!bit) break;
            nonzero = 1;
            dec_len = i + 1;
        }
        if (c->encode) {
            REGIME(RG_AC_LEN11, length == 11);
            REGIME(RG_REFUSE_AC, length > 11);
            if (length > 11) { c->err = LO_COEFFICIENT_OUT_OF_RANGE; return; }
            nonzero = coef != 0;
        } else {
            length = dec_len;
        }
        if (nonzero) {
            int min_thr = qt->min_noise_threshold[coord];
            int16_t v16 = (int16_t)prior; /* sign_array_8, model.hh:1114-1122: int16 truncation of best_prior */
            REGIME(RG_SIGN_CTX_INT16, v16 != prior);
            int sctx = v16 == 0 ? 0 : (v16 > 0 ? 1 : 2);
            int sbit = code_bit(c, &c->model->sign[ci][sctx][bsr], coef >= 0);
            int neg = !sbit;
            int val = 1 << (length - 1);
            --ne;
            if (length > 1) {
                int i = length - 2;
                if (i >= min_thr) {
                    uint16_t ctx_abs = (uint16_t)iabs(prior); /* residual_thresh_array, model.hh:1072-1088 */
                    REGIME(RG_THR_CTX_MASK, ctx_abs != (int64_t)iabs(prior));
                    REGIME(RG_THR_CTX_CAP255, (ctx_abs >> min_thr) > 255);
                    Branch *thr = c->model->res_thresh[ci][imin(ctx_abs >> min_thr, 255)][imin(length - min_thr, 7)];
                    unsigned so = 1;
                    for (; i >= min_thr; --i) {
                        int bit = code_bit(c, &thr[so], (abs_coef >> i) & 1);
                        val |= bit << i;
                        so = (so << 1) | (unsigned)bit;
                        REGIME(RG_THR_SO_SAT127, so > 127);
                        if (so > 127) so = 127;
                    }
                }
                Branch *res = c->model->res_noise[ci][coord][nzbin]; /* residual_noise_array_x, model.hh:537-551 */
                for (; i >= 0; --i) {
                    int bit = code_bit(c, &res[i], (abs_coef >> i) & 1);
                    val |= bit << i;
                }
            }
            if (!c->encode) coef = (int16_t)(neg ? -val : val);
        }
        if (!c->encode) here_mut[aligned_off + lane] = coef;
    }
}

/* serialize_tokens (encoder.cc:194-402) / parse_tokens (decoder.cc:167-318) */
static void code_block(Codec *c, int cmp, const BlockCtx *b, int16_t *here_mut) {
    const int ci = cmp == 0 ? 0 : 1; /* color_index, model.hh:373-382 */
    const QuantTables *qt = &c->qt[cmp];
    if (!c->encode) memset(here_mut, 0, 128);
    Branch(*nzp)[32] = (Branch(*)[32])nz7x7_slice(c, ci, b);
    int nz = 0;
    if (c->encode) { /* recalculate_coded_length, aligned_block.hh:132-148 */
        for (int i = 0; i < 49; ++i) nz += b->here[i] != 0;
        b->ns_here->nz = (uint8_t)nz; /* vp8_encoder.cc:103 */
    }
    int so_far = 0, nz_dec = 0;
    for (int idx = 5; idx >= 0; --idx) {
        int bit = code_bit(c, &nzp[idx][so_far], (nz >> idx) & 1);
        nz_dec |= bit << idx;
        so_far = (so_far << 1) | bit;
    }
    if (!c->encode) nz = nz_dec;
    if (nz > 49) { c->err = LO_STREAM_INCONSISTENT; return; }
    int eob_x = 0, eob_y = 0, left_nz = nz;
    for (int zz = 0; zz < 49 && left_nz; ++zz) {
        int coord = k_aligned_to_raster[zz]; /* == unzigzag49[zz] */
        int bx = coord & 7, by = coord >> 3;
        int16_t prior = aavrg(b, zz);
        int nzbin = k_nonzero_to_bin[left_nz];
        int bsr = bit_length((uint32_t)imin(iabs(prior), 1023));
        REGIME(RG_BSR_CAP1023, iabs(prior) > 1023);
        Branch *exp = c->model->exp7x7[ci][nzbin][zz][bsr];
        int16_t coef = c->encode ? b->here[zz] : 0;
        uint16_t abs_coef = (uint16_t)iabs(coef);
        int length = bit_length(abs_coef), dec_len = 0, nonzero = 0;
        for (int i = 0; i < 11; ++i) {
            int bit = code_bit(c, &exp[i], length != i);
            if (!bit) break;
            nonzero = 1;
            dec_len = i + 1;
        }
        if (c->encode) {
            REGIME(RG_AC_LEN11, length == 11);
            REGIME(RG_REFUSE_AC, length > 11);
            if (length > 11) { c->err = LO_COEFFICIENT_OUT_OF_RANGE; return; }
            nonzero = length != 0;
        } else {
            length = dec_len;
        }
        if (nonzero) {
            int sbit = code_bit(c, &c->model->sign[ci][0][0], coef >= 0);
            int neg = !sbit;
            --left_nz;
            eob_x = imax(eob_x, bx);
            eob_y = imax(eob_y, by);
            int val = 1 << (length - 1);
            if (length > 1) {
                Branch *res = c->model->res_noise[ci][coord][nzbin];
                for (int i = length - 2; i >= 0; --i) {
                    int bit = code_bit(c, &res[i], (abs_coef >> i) & 1);
                    val |= bit << i;
                }
            }
            if (!c->encode) coef = (int16_t)(neg ? -val : val);
        }
        if (!c->encode) here_mut[zz] = coef;
    }
    code_one_edge(c, cmp, ci, b, here_mut, 1, nz, eob_x);
    if (c->err) return;
    code_one_edge(c, cmp, ci, b, here_mut, 0, nz, eob_y);
    if (c->err) return;

    int16_t pix[64];
    int unc = 0, unc2 = 0;
    int pred = adv_predict_dc_pix(b, qt, pix, &unc, &unc2);
    int16_t coef = 0;
    if (c->encode) {
        int adv = adv_unpredict(b->here[49], 0, pred);
        if (b->here[49] != adv_unpredict((int16_t)adv, 1, pred)) { ++g_regime[RG_REFUSE_DC]; c->err = LO_COEFFICIENT_OUT_OF_RANGE; return; }
        coef = (int16_t)adv;
    }
    {
        uint16_t abs_coef = (uint16_t)iabs(coef);
        int length = bit_length(abs_coef), dec_len = 0, nonzero = 0;
        int len_mxm = bit_length((uint16_t)iabs(unc));   /* uint16bit_length(abs(uncertainty)), encoder.cc:322 */
        int len_off = bit_length((uint16_t)iabs(unc2));
        REGIME(RG_LEN_MXM_CAP11, len_mxm > 11);
        Branch *exp = c->model->exp_dc[imin(len_mxm, 11)][imin(len_off, 16)]; /* model.hh:520-529 */
        for (int i = 0; i < 11; ++i) {
            int bit = code_bit(c, &exp[i], length != i);
            if (!bit) break;
            nonzero = 1;
            dec_len = i + 1;
        }
        if (c->encode) {
            REGIME(RG_REFUSE_DC_LEN, length > 11);
            if (length > 11) { c->err = LO_COEFFICIENT_OUT_OF_RANGE; return; }
            nonzero = length != 0;
        } else {
            length = dec_len;
        }
        if (nonzero) {
            int sctx = unc2 >= 0 ? (unc2 == 0 ? 3 : 2) : 1; /* sign_array_dc, model.hh:1100-1109 */
            int sbit = code_bit(c, &c->model->sign[ci][0][sctx], coef >= 0);
            int neg = !sbit;
            int val = 1 << (length - 1);
            if (length > 1) {
                Branch *res = c->model->res_noise_dc[imin(len_mxm, 11)]; /* residual_array_dc, model.hh:530-536 */
                for (int i = length - 2; i >= 0; --i) {
                    int bit = code_bit(c, &res[i], (abs_coef >> i) & 1);
                    val |= bit << i;
                }
            }
            if (!c->encode) coef = (int16_t)(neg ? -val : val);
        }
    }
    int16_t dc;
    if (c->encode) {
        dc = b->here[49];
    } else {
        dc = (int16_t)adv_unpredict(coef, 1, pred); /* decoder.cc:305-309 */
        here_mut[49] = dc;
        b->ns_here->nz = (uint8_t)nz; /* decoder.cc:310 */
    }
    ns_set_edges(b->ns_here, pix, qt->q, dc);
}

/* ------------------------------------------------------------------ row / segment driver */
typedef struct { int luma_y, component, curr_y, skip, done; } RowSpec;

/* LeptonCodec_row_spec_from_index, src/lepton/lepton_codec.hh:41-100 */
static RowSpec row_spec_from_index(uint32_t idx, const lo_geometry *g) {
    uint32_t mult[3] = {0, 0, 0}, mcu_multiple = 0;
    for (int i = 0; i < 3; ++i) {
        uint32_t h = i < g->ncmp ? (uint32_t)g->bcv[i] : 0;
        mult[i] = h / (uint32_t)g->mcuv;
        mcu_multiple += mult[i];
    }
    uint32_t mcu_row = idx / mcu_multiple;
    uint32_t place = idx - mcu_row * mcu_multiple;
    RowSpec r = {0, 3, 0, 0, 0};
    r.luma_y = (int)(mcu_row * mult[0]);
    for (int i = 2;; --i) {
        if (place < mult[i]) {
            r.component = i;
            r.curr_y = (int)(mcu_row * mult[i] + place);
            uint32_t maxh_i = i < g->ncmp ? (uint32_t)g->trunc_bcv[i] : 0;
            if (r.curr_y >= (int)maxh_i) {
                r.skip = 1;
                r.done = 1;
                for (int j = 0; j < 2; ++j) {
                    uint32_t maxh_j = j < g->ncmp ? (uint32_t)g->trunc_bcv[j] : 0;
                    if (mcu_row * mult[j] < maxh_j) r.done = 0;
                }
            }
            if (i == 0) r.luma_y = r.curr_y;
            break;
        }
        place -= mult[i];
        if (i == 0) { r.skip = 1; r.done = 1; break; }
    }
    return r;
}

/* process_row (vp8_encoder.cc:83-154) / ThreadState::decode_row (lepton_codec.cc:7-47) */
static void code_row(Codec *c, int cmp, int y, int top_row) {
    const lo_geometry *g = c->g;
    int w = g->bch[cmp];
    int16_t *plane = c->planes[cmp];
    NeighborSummary *here_row = c->ns[cmp] + ((y & 1) ? w : 0);
    NeighborSummary *above_row = c->ns[cmp] + ((y & 1) ? 0 : w);
    for (int x = 0; x < w; ++x) {
        /* model selection: vp8_encoder.cc:294-339 (corner/top on a segment's first row of the component,
         * midleft/middle/midright afterwards, width_one :232-237) */
        int left_present = x > 0;
        int above_present = !top_row;
        BlockCtx b;
        int16_t *here = plane + ((size_t)y * w + x) * 64;
        b.here = here;
        b.left = left_present ? here - 64 : NULL;
        b.above = above_present ? here - (size_t)w * 64 : NULL;
        b.above_left = (left_present && above_present) ? here - (size_t)w * 64 - 64 : NULL;
        b.ns_here = here_row + x;
        b.ns_left = left_present ? here_row + x - 1 : NULL;
        b.ns_above = above_present ? above_row + x : NULL;
        code_block(c, cmp, &b, here);
        if (c->err) return;
        if (c->encode && c->bw.overflow) { c->err = LO_OUTPUT_OVERFLOW; return; }
        /* early-out on truncated images: vp8_encoder.cc:110-113,133-135 / lepton_codec.cc:22-24,33-35;
         * not applied after the right-most block (vp8_encoder.cc:151) */
        if (x + 1 < w || w == 1) {
            uint32_t offset = (uint32_t)((size_t)y * w + x + 1);
            if (x + 1 < w && offset >= (uint32_t)g->trunc_bc[cmp]) return;
            if (w == 1 && offset >= (uint32_t)g->trunc_bc[cmp]) return;
        }
    }
}

/* process_row_range (vp8_encoder.cc:239-445) / vp8_decode_thread (lepton_codec.cc:266-309) */
static int code_segment(Codec *c, int min_y, int max_y, int is_last) {
    int top[3] = {1, 1, 1};
    uint32_t index = 0;
    for (;;) {
        RowSpec r = row_spec_from_index(index++, c->g);
        if (r.done) break;
        if (r.luma_y >= max_y && !is_last) break;
        if (r.skip) continue;
        if (r.luma_y < min_y) continue;
        int t = top[r.component];
        top[r.component] = 0;
        code_row(c, r.component, r.curr_y, t);
        if (c->err) return c->err;
    }
    return 0;
}

static int codec_init(Codec *c, const lo_geometry *g, int16_t *const planes[3], int encode) {
    lo_init_tables();
    memset(c, 0, sizeof(*c));
    c->g = g;
    c->encode = encode;
    if (g->ncmp < 1 || g->ncmp > 3 || g->mcuv <= 0) return LO_ASSERTION_FAILURE;
    for (int i = 0; i < g->ncmp; ++i) {
        int e = quant_tables_init(&c->qt[i], g->q_zigzag[i]);
        if (e && encode) return e; /* decoder (filetype==LEPTON) skips the zero check, model.hh:257 */
        c->planes[i] = planes[i];
        c->ns[i] = (NeighborSummary *)calloc((size_t)g->bch[i] * 2 + 1, sizeof(NeighborSummary));
    }
    c->model = (Model *)malloc(sizeof(Model));
    model_reset(c->model);
    return 0;
}
static void codec_free(Codec *c) {
    for (int i = 0; i < 3; ++i) free(c->ns[i]);
    free(c->model);
}

/* Encode one thread-segment [min_y, max_y) of luma rows into its own bool-coder stream.
 * Returns a reference ExitCode value (0 ok).  ndecisions (optional) = number of put() calls. */
int lo_encode_segment(const lo_geometry *g, const int16_t *const planes[3], int min_y, int max_y, int is_last,
                      uint8_t *out, size_t cap, size_t *out_len, uint64_t *ndecisions) {
    Codec c;
    int e = codec_init(&c, g, (int16_t *const *)planes, 1);
    if (e) { codec_free(&c); return e; }
    if (cap < 64) { codec_free(&c); return LO_OUTPUT_OVERFLOW; }
    bw_start(&c.bw, out, cap - 8);
    e = code_segment(&c, min_y, max_y, is_last);
    if (!e) {
        bw_stop(&c.bw);
        if (c.bw.overflow) e = LO_OUTPUT_OVERFLOW;
        *out_len = c.bw.pos;
    }
    if (ndecisions) *ndecisions = c.ndecisions;
    codec_free(&c);
    return e;
}

/* Decode one thread-segment stream back into the coefficient planes (rows of this segment only). */
int lo_decode_segment(const lo_geometry *g, int16_t *const planes[3], int min_y, int max_y, int is_last,
                      const uint8_t *in, size_t in_len, uint64_t *ndecisions) {
    Codec c;
    int e = codec_init(&c, g, planes, 0);
    if (e) { codec_free(&c); return e; }
    br_init(&c.br, in, in_len);
    e = code_segment(&c, min_y, max_y, is_last);
    if (ndecisions) *ndecisions = c.ndecisions;
    codec_free(&c);
    return e;
}

/* The bool coder alone: vpx_start_encode, one vpx_write per token, vpx_stop_encode.  Token k = prob | bit << 8 (the
 * layout kernel A writes).  Returns 0, or LO_OUTPUT_OVERFLOW when the stream (plus 2 bytes of room) does not fit `cap`;
 * then *out_len = 0 and the bytes in `out` are meaningless. */
int lo_bool_encode(const uint16_t *tokens, size_t n, uint8_t *out, size_t cap, size_t *out_len) {
    *out_len = 0;
    if (cap < 8) return LO_OUTPUT_OVERFLOW;
    BoolWriter w;
    bw_start(&w, out, cap);
    for (size_t i = 0; i < n && !w.overflow; ++i) bw_write(&w, (tokens[i] >> 8) & 1, tokens[i] & 0xff);
    if (w.overflow) return LO_OUTPUT_OVERFLOW;
    bw_stop(&w);
    if (w.overflow) return LO_OUTPUT_OVERFLOW;
    *out_len = w.pos;
    return 0;
}
void lo_bool_counts(uint64_t out[3]) { out[0] = g_bw_walk_max; out[1] = g_bw_walk_long; out[2] = g_bw_stop_zero; }
void lo_bool_counts_reset(void) { g_bw_walk_max = g_bw_walk_long = g_bw_stop_zero = 0; }

size_t lo_model_bytes(void) { return sizeof(Model); }

/* regime counters: names, values (since the last reset), reset */
int lo_regime_count(void) { return RG_COUNT; }
const char *lo_regime_name(int i) { return i >= 0 && i < RG_COUNT ? k_regime_names[i] : NULL; }
uint64_t lo_regime_value(int i) { return i >= 0 && i < RG_COUNT ? g_regime[i] : 0; }
void lo_regime_reset(void) { memset(g_regime, 0, sizeof(g_regime)); }
