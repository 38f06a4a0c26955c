// lep_decode.cu -- sm_90a decode kernel: per-segment VP8 bool-coder streams -> coefficient planes.
//
// Decoding is a true serial dependency chain: every context index depends on previously decoded values
// (remaining non-zero count, exponent so far, neighbours in the same block), so unlike the encoder the
// symbol stream cannot be produced ahead of the coder.  One warp owns one thread-segment; the bool decoder
// state (vpx_reader, src/vp8/decoder/boolreader.hh:184-258,376-416) and the token grammar
// (parse_tokens, src/vp8/decoder/decoder.cc:167-318) run warp-uniform, while the work that IS data-parallel
// is spread over the lanes: the 49 aavrg priors, the 14 Lakhani edge predictors, the 8x8 IDCT, the DC
// estimate reductions and the coalesced 128-byte block loads/stores.
#include "lep_common.cuh"
#include "lep_predict.cuh"

namespace lepb200 {

constexpr int DEC_WARPS_PER_CTA = 4;

struct DecWarpSmem {
    int16_t rast[3][64];      // raster-order copies: cur / left ping-pong, above
    int32_t tmp[64];
    int16_t pix[64];
};
struct DecShared {
    uint32_t rcp[512];
    DecWarpSmem w[DEC_WARPS_PER_CTA];
};

struct BoolReader {
    unsigned long long value;
    uint32_t range;
    int count;
    const uint8_t* p;
    const uint8_t* end;
};

// vpx_reader_fill (boolreader.hh:184-258): big-endian refill, zero bits past the end of the stream.
__device__ __forceinline__ void br_fill(BoolReader& r) {
    int shift = 64 - 8 - (r.count + 8);
    while (shift >= 0) {
        unsigned long long byte = (r.p < r.end) ? (unsigned long long)__ldg(r.p) : 0ull;
        r.p++;
        r.value |= byte << shift;
        r.count += 8;
        shift -= 8;
    }
}

// The kernel's two entropy coders share one interface: coder_init (state before the first decision), coder_read (one decision
// at an 8-bit probability) and coder_pos (where the reader is in the stream).
__device__ __forceinline__ void coder_init(BoolReader& r, const uint8_t* p, uint32_t len) {
    r.value = 0; r.count = -8; r.range = 255;
    r.p = p; r.end = p + len;
    br_fill(r);
    // marker bit at p = 128 (boolreader.cc:26-35); no model involved
    uint32_t split = (r.range * 128u + 128u) >> 8;
    unsigned long long bigsplit = (unsigned long long)split << 56;
    uint32_t bit = r.value >= bigsplit;
    uint32_t range = bit ? r.range - split : split;
    if (bit) r.value -= bigsplit;
    int shift = __clz(range) - 24;
    r.range = range << shift; r.value <<= shift; r.count -= shift;
}
// vpx_read (boolreader.hh:376-416)
__device__ __forceinline__ uint32_t coder_read(BoolReader& r, uint32_t prob) {
    uint32_t split = (r.range * prob + (256 - prob)) >> 8;
    if (r.count < 0) br_fill(r);
    const uint32_t bit = (uint32_t)(r.value >> 56) >= split;          // value >= split << 56  <=>  top byte >= split
    uint32_t range = bit ? r.range - split : split;
    if (bit) r.value -= (unsigned long long)split << 56;
    int shift = __clz(range) - 24;
    r.range = range << shift;
    r.value <<= shift;
    r.count -= shift;
    return bit;
}
__device__ __forceinline__ const uint8_t* coder_pos(const BoolReader& r) { return r.p; }
// the bool coder's model: probability and record_obs_and_update (branch.hh:82-100); a plain increment unless a count is
// about to saturate (or the word is the special state)
__device__ __forceinline__ uint32_t coder_prob(const BoolReader&, uint32_t w, const uint32_t* rcp) { return branch_prob(w, rcp); }
__device__ __forceinline__ uint32_t coder_model_word(const BoolReader&, uint32_t w, uint32_t bit) {
    const bool plain = (w & 0xffu) < 254u && (w >> 8) < 254u;
    return plain ? w + (bit ? 0x100u : 1u) : branch_update(w, bit);
}

// ANSBoolReader (ans_bool_reader.hh:75-108, rans64.hh:108-139): two 64-bit rANS states that take turns, 8-bit probabilities,
// the stream read as little-endian 32-bit words, at most one per decision, zero past the end (fill()).
struct AnsReader {
    unsigned long long x0, x1;        // the state of the next decision, the one after it
    const uint8_t* p;                 // next word
    const uint8_t* end;
};
// the word at p: streams start 16-byte aligned and their slots are readable up to the next 16 bytes
__device__ __forceinline__ uint32_t ans_word(const uint8_t* p, const uint8_t* end) {
    const long long rem = end - p;
    if (rem <= 0) return 0u;
    uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(p));
    if (rem < 4) w &= 0xffffffffu >> (8 * (4 - (int)rem));             // the bytes behind the stream read as zero
    return w;
}
// Rans64DecInit twice: words 0-1 and 2-3, low word first
__device__ __forceinline__ void coder_init(AnsReader& r, const uint8_t* p, uint32_t len) {
    r.p = p; r.end = p + len;
    r.x0 = (unsigned long long)ans_word(r.p, r.end) | (unsigned long long)ans_word(r.p + 4, r.end) << 32;
    r.x1 = (unsigned long long)ans_word(r.p + 8, r.end) | (unsigned long long)ans_word(r.p + 12, r.end) << 32;
    r.p += 16;
}
// ANSBoolReader::get: Rans64DecGet / Rans64DecAdvance at scale 8 on the first state, which then becomes the second
__device__ __forceinline__ uint32_t coder_read(AnsReader& r, uint32_t prob) {
    unsigned long long x = r.x0;
    r.x0 = r.x1;
    const uint32_t cf = (uint32_t)x & 255u;
    const uint32_t bit = cf >= prob;
    const uint32_t start = bit ? prob : 0u;
    const uint32_t freq = (prob ^ (0u - bit)) + (bit | (bit << 8));      // bit ? 256 - prob : prob
    x = (unsigned long long)freq * (x >> 8) + cf - start;
    if (x < (1ull << 31)) { x = (x << 32) | ans_word(r.p, r.end); r.p += 4; }
    r.x1 = x;
    return bit;
}
__device__ __forceinline__ const uint8_t* coder_pos(const AnsReader& r) { return r.p; }
// the rANS coder's model (adv_record_obs_and_update, lep_common.cuh)
__device__ __forceinline__ uint32_t coder_prob(const AnsReader&, uint32_t w, const uint32_t* rcp) { return branch_prob_ans(w, rcp); }
__device__ __forceinline__ uint32_t coder_model_word(const AnsReader&, uint32_t w, uint32_t bit) { return branch_update_ans(w, bit); }

template <class Reader> struct Decoder {
    Reader br;
    uint16_t* model;
    const uint32_t* rcp;
    unsigned long long ndec;
};

// VPXBoolReader::get (vpx_bool_reader.hh:45-57) / ANSBoolReader::get (ans_bool_reader.hh:87-108) = one decision + the
// branch's update (record_obs_and_update / adv_record_obs_and_update)
template <class Reader> __device__ __forceinline__ uint32_t dec_get(Decoder<Reader>& d, uint32_t addr) {
    uint32_t w = d.model[addr];
#ifdef LEPB200_EMU
    __syncwarp();      // CPU warp emulator (tests/emu) only: lanes run one after the other there, so every lane must have
                       // read the count before the first one writes it back; on the device the converged warp does that anyway
#endif
    uint32_t prob = coder_prob(d.br, w, d.rcp);
    const uint32_t bit = coder_read(d.br, prob);
    d.model[addr] = (uint16_t)coder_model_word(d.br, w, bit);      // every lane stores the same value (one transaction)
    d.ndec++;
    return bit;
}

// exponent unary + sign + residual bits of one coefficient (decoder.cc:212-240); returns the signed value
template <class Reader> __device__ __forceinline__ int dec_coef_plain(Decoder<Reader>& d, uint32_t exp_addr, uint32_t sign_addr, uint32_t res_addr, int& len_out) {
    int len = 0;
    while (len < 11) { if (!dec_get(d, m_exp_word(exp_addr, len))) break; ++len; }
    len_out = len;
    if (len == 0) return 0;
    bool neg = !dec_get(d, sign_addr);
    int val = 1 << (len - 1);
    for (int i = len - 2; i >= 0; --i) val |= (int)dec_get(d, res_addr + i) << i;
    return neg ? -val : val;
}

#ifndef LEPB200_DEC_MINBLOCKS
#define LEPB200_DEC_MINBLOCKS 5
#endif
// Reader: BoolReader (container versions 1, 2, 4) or AnsReader (version 3); every segment of a launch uses that coder
template <class Reader = BoolReader>
__global__ void __launch_bounds__(DEC_WARPS_PER_CTA * 32, LEPB200_DEC_MINBLOCKS)
lep_decode_kernel(const ImageDesc* __restrict__ images, SegDesc* __restrict__ segs, int nseg, const int* __restrict__ order,
                  int* __restrict__ work_counter, uint16_t* __restrict__ model_pool, uint8_t* __restrict__ row_pool,
                  size_t row_pool_stride) {
    __shared__ DecShared sm;
    const int lane = lane_id();
    const int warp_in_cta = threadIdx.x >> 5;
    const int gwarp = blockIdx.x * DEC_WARPS_PER_CTA + warp_in_cta;
    for (int i = threadIdx.x; i < 512; i += blockDim.x) sm.rcp[i] = i < 2 ? 0u : (uint32_t)((0x100000000ull + i - 1) / i);
    __syncthreads();
    DecWarpSmem& ws = sm.w[warp_in_cta];
    const int r0 = c_aligned_to_raster[2 * lane], r1 = c_aligned_to_raster[2 * lane + 1];   // once: per-lane constant-memory indices serialise
    uint16_t* model = model_pool + (size_t)gwarp * M_TOTAL;
    uint8_t* rowbuf = row_pool + (size_t)gwarp * row_pool_stride;

    for (;;) {
        int job = 0;
        if (lane == 0) job = atomicAdd(work_counter, 1);
        job = __shfl_sync(FULL, job, 0);
        if (job >= nseg) break;
        const int sidx = order[job];
        SegDesc& sd = segs[sidx];
        const ImageDesc& g = images[sd.image];
        if (sd.status != ST_OK) continue;          // rejected on the host (e.g. zero quantiser, model.hh:257-262)
        {
            uint4* m4 = reinterpret_cast<uint4*>(model);
            const uint4 z = make_uint4(0, 0, 0, 0);
            for (uint32_t i = lane; i < M_TOTAL / 8; i += 32) LEP_ST_STREAM(m4, i, z);
        }
        __syncwarp();

        Decoder<Reader> d;
        d.model = model; d.rcp = sm.rcp; d.ndec = 0;
        coder_init(d.br, reinterpret_cast<const uint8_t*>(sd.stream), sd.cap);

        // per-component row buffers (offsets kept as scalars: arrays indexed by the component would live in local memory)
        const int bw0 = g.bch[0], bw1 = g.ncmp > 1 ? g.bch[1] : 0, bw2 = g.ncmp > 2 ? g.bch[2] : 0;
        const size_t nz_base = (size_t)(bw0 + bw1 + bw2) * 16;
        const int nzs0 = (bw0 + 15) & ~15, nzs1 = (bw1 + 15) & ~15;

        int status = ST_OK;
        uint32_t top_mask = 7u;
        uint32_t index = 0;
        for (;;) {
            RowSpec rs = row_spec_from_index(index++, g);
            if (rs.done) break;
            if (rs.luma_y >= sd.max_y && !sd.is_last) break;
            if (rs.skip) continue;
            if (rs.luma_y < sd.min_y) continue;
            const int c = rs.component, y = rs.curr_y;
            const bool has_above = !((top_mask >> c) & 1u);
            top_mask &= ~(1u << c);
            const int ci = c == 0 ? 0 : 1;
            const int w = g.bch[c];
            uint32_t* plane = reinterpret_cast<uint32_t*>(g.plane[c]);
            uint32_t* rowp = plane + (size_t)y * w * 32;
            const uint32_t* abovep = rowp - (size_t)w * 32;
            const uint16_t* q = g.q[c];
            const int q0 = q[0];
            int16_t* redge = reinterpret_cast<int16_t*>(rowbuf + (size_t)(c == 0 ? 0 : (c == 1 ? bw0 : bw0 + bw1)) * 16);
            uint8_t* rnz = rowbuf + nz_base + (c == 0 ? 0 : (c == 1 ? nzs0 : nzs0 + nzs1));

            uint32_t abv = has_above ? LEP_LD_LAST(abovep, lane) : 0u;
            uint32_t left = 0, aleft = 0;
            int left_v = 0, nz_left = 0, pp = 0;
            for (int x = 0; x < w; ++x) {
                const bool has_left = x > 0;
                uint32_t nabv = 0;
                if (has_above && x + 1 < w) nabv = LEP_LD_LAST(abovep, (size_t)(x + 1) * 32 + lane);
                ws.rast[2][r0] = (int16_t)h_lo(abv); ws.rast[2][r1] = (int16_t)h_hi(abv);
                int16_t* rcur = ws.rast[pp];
                const int16_t* rleft = ws.rast[pp ^ 1];
                const int16_t* rabove = ws.rast[2];

                // ---- (i) 7x7 non-zero count
                const int nz_above = has_above ? (int)rnz[x] : 0;
                int nz = 0;
                {
                    int ctx = 0;
                    if (has_above && !has_left) ctx = (nz_above + 1) / 2;
                    else if (has_left && !has_above) ctx = (nz_left + 1) / 2;
                    else if (has_left && has_above) ctx = (nz_above + nz_left + 2) / 4;
                    const int bin = c_nonzero_to_bin[ctx];
                    int prefix = 0;
                    for (int idx = 5; idx >= 0; --idx) {
                        uint32_t b = dec_get(d, m_nz7(ci, bin, idx, prefix));
                        nz |= (int)b << idx;
                        prefix = (prefix << 1) | (int)b;
                    }
                }
                if (nz > 49) { status = ST_STREAM_INCONSISTENT; break; }
                // ---- (ii) 7x7 coefficients
                const int pr0 = aavrg16(h_lo(left), h_lo(abv), h_lo(aleft), has_left, has_above);
                const int pr1 = aavrg16(h_hi(left), h_hi(abv), h_hi(aleft), has_left, has_above);
                int lo = 0, hi = 0;       // this lane's two coefficients of the block being decoded
                int eobx = 0, eoby = 0, left_nz = nz;
                for (int zz = 0; zz < 49 && left_nz > 0; ++zz) {
                    const int prior = __shfl_sync(FULL, (zz & 1) ? pr1 : pr0, zz >> 1);
                    const int bin = c_nonzero_to_bin[left_nz];
                    const int bsr = bitlen((uint32_t)min(iabs(prior), 1023));
                    const int coord = c_aligned_to_raster[zz];
                    int len;
                    const int v = dec_coef_plain(d, m_exp7(ci, bin, zz, bsr), m_sign(ci, 0, 0), m_resn(ci, coord, bin), len);
                    if (len) {
                        --left_nz;
                        eobx = max(eobx, coord & 7); eoby = max(eoby, coord >> 3);
                        if (lane == (zz >> 1)) { if (zz & 1) hi = v; else lo = v; }
                    }
                }
                // raster copy of the 7x7 part (edges and DC still zero) for the edge predictors
                rcur[r0] = (int16_t)lo; rcur[r1] = (int16_t)hi;
                __syncwarp();
                // ---- (iii) edges
                {
                    const bool is_h = lane < 7, is_v = lane >= 8 && lane < 15;
                    const int k = is_h ? lane + 1 : lane - 7;
                    int prior_l = 0;
                    if (is_h && has_above) prior_l = lak_pred(rcur, rabove, g.icos_x[c] + k * 8, k, 8);
                    if (is_v && has_left) prior_l = lak_pred(rcur, rleft, g.icos_y[c] + k * 8, 8 * k, 1);
                    __syncwarp();
                    for (int vert = 0; vert < 2; ++vert) {
                        const int eob = vert ? eoby : eobx;
                        int ne = 0, prefix = 0;
                        for (int i = 2; i >= 0; --i) {
                            uint32_t b = dec_get(d, m_nze(vert, ci, eob, (nz + 3) / 7, i, prefix));
                            ne |= (int)b << i;
                            prefix = (prefix << 1) | (int)b;
                        }
                        for (int ln = 0; ln < 7 && ne > 0; ++ln) {
                            const int kk = ln + 1;
                            const int coord = vert ? 8 * kk : kk;
                            const int zig15 = vert ? 7 + ln : ln;
                            const int prior = __shfl_sync(FULL, prior_l, vert ? 8 + ln : ln);
                            const int bsr = bitlen((uint32_t)min(iabs(prior), 1023));
                            const uint32_t ea = m_expx(ci, ne, zig15, bsr);
                            int len = 0;
                            while (len < 11) { if (!dec_get(d, m_exp_word(ea, len))) break; ++len; }
                            int v = 0;
                            if (len) {
                                const int p16 = (int)(int16_t)prior;
                                const int sctx = p16 == 0 ? 0 : (p16 > 0 ? 1 : 2);
                                const bool neg = !dec_get(d, m_sign(ci, sctx, bsr));
                                const int ne0 = ne;
                                --ne;
                                int val = 1 << (len - 1);
                                if (len > 1) {
                                    const int min_thr = g.min_thr[c][coord];
                                    int i = len - 2;
                                    if (i >= min_thr) {
                                        const int ctx_abs = iabs(prior) & 0xffff;
                                        const uint32_t ta = m_thr(ci, min(ctx_abs >> min_thr, 255), min(len - min_thr, 7));
                                        uint32_t so = 1;
                                        for (; i >= min_thr; --i) {
                                            uint32_t b = dec_get(d, ta + so);
                                            val |= (int)b << i;
                                            so = min((so << 1) | b, 127u);
                                        }
                                    }
                                    const uint32_t ra = m_resn(ci, coord, ne0);
                                    for (; i >= 0; --i) val |= (int)dec_get(d, ra + i) << i;
                                }
                                v = neg ? -val : val;
                                const int aidx = (vert ? 57 : 50) + ln;           // aligned index of this edge coefficient
                                if (lane == (aidx >> 1)) { if (aidx & 1) hi = v; else lo = v; }
                            }
                        }
                    }
                }
                // raster copy now complete except DC (forced to zero by the IDCT anyway)
                rcur[r0] = (int16_t)lo; rcur[r1] = (int16_t)hi;
                __syncwarp();
                // ---- (iv) DC
                warp_idct_sans_dc(rcur, q, ws.tmp, ws.pix, lane);
                int above_h = 0;
                if (has_above && lane >= 8 && lane < 16) above_h = redge[(size_t)x * 8 + (lane - 8)];
                DcPred dp = warp_predict_dc(ws.pix, left_v, above_h, has_left, has_above, q0, lane);
                int dc;
                {
                    const int lm = min(bitlen((uint32_t)iabs(dp.unc) & 0xffff), 11), lo16 = min(bitlen((uint32_t)iabs(dp.unc2) & 0xffff), 16);
                    const int sctx = dp.unc2 >= 0 ? (dp.unc2 == 0 ? 3 : 2) : 1;
                    int len;
                    const int v = dec_coef_plain(d, m_expdc(lm, lo16), m_sign(ci, 0, sctx), m_resdc(lm), len);
                    dc = (int)(int16_t)adv_unpredict((int)(int16_t)v, true, dp.pred);      // decoder.cc:305-309
                }
                if (lane == 24) hi = dc;                                                    // aligned index 49
                // ---- (v) neighbour summary + store the block
                const int edge = edge_pixel(ws.pix, q0, dc, lane);
                if (lane >= 8 && lane < 16) redge[(size_t)x * 8 + (lane - 8)] = (int16_t)edge;
                if (lane == 0) rnz[x] = (uint8_t)nz;
                left_v = edge;
                nz_left = nz;
                const uint32_t curw = ((uint32_t)lo & 0xffffu) | ((uint32_t)hi << 16);
                rowp[(size_t)x * 32 + lane] = curw;
                if (lane == 24) rcur[0] = (int16_t)dc;     // keep the raster copy complete for the next block's predictors
                __syncwarp();

                if (x + 1 < w && (uint32_t)((size_t)y * w + x + 1) >= (uint32_t)g.trunc_bc[c]) break;
                aleft = abv; left = curw; abv = nabv; pp ^= 1;
            }
            if (status != ST_OK) break;
        }
        if (lane == 0) {
            sd.status = status;
            sd.len = (uint32_t)(coder_pos(d.br) - reinterpret_cast<const uint8_t*>(sd.stream));
            sd.ndecisions_lo = (uint32_t)d.ndec;
            sd.ndecisions_hi = (uint32_t)(d.ndec >> 32);
        }
        __syncwarp();
    }
}

}  // namespace lepb200
