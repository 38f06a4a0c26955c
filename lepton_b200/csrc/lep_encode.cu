// lep_encode.cu -- sm_90a encode kernels: coefficient planes -> per-segment VP8 bool-coder streams.
//
// Work decomposition (new; the reference runs one CPU thread per segment, src/lepton/vp8_encoder.cc:239-445):
//   * persistent grid, one WARP per Lepton thread-segment, segments pulled from a global work queue
//     (largest first), the warp's 1.58 MB probability model zero-filled by the warp itself;
//   * kernel A (lep_encode_kernel) codes TWO blocks (x, x + 1) per iteration in two phases
//       1. lane-parallel SYMBOLISATION.  Nothing in the encoder's context computation depends on coder state
//          (SURVEY.md section 7, hard part 1), so the warp computes, for both blocks, the neighbour priors /
//          context bins of all coefficients (each lane owns two coefficients of each block: one 32-bit word of the
//          128-byte AlignedBlock) and -- with lanes 0..15 serving block x and 16..31 block x + 1 -- the lane-sparse
//          parts at double width: 8x8 IDCT (8 lanes per block), DC prediction (16), Lakhani edge predictors and
//          edge counts (15).  Every coded coefficient leaves one 16-byte ITEM in shared memory;
//       2. the FLUSH expands the items to (branch index, bit) decisions 32 at a time, one per lane: parallel 16-bit
//          loads of the adaptive counts (next step's words prefetched), same-branch conflicts resolved in queue
//          order in closed form (__match_any_sync + popcounts), probabilities computed per lane, counts written
//          back; the resulting (probability, bit) TOKENS (16 bits each) go to the segment's token stream in HBM
//          with coalesced 64-byte stores;
//   * kernel B (lep_rangecode_kernel) runs the serial RANGE CODER chain (vpx_write,
//     src/vp8/encoder/boolwriter.hh:48-118) with one THREAD per segment: the chain needs no memory-dependent
//     loads any more, so 32 segments advance per warp instruction instead of one;
//   * lep_count_kernel / lep_token_offsets_kernel size the token streams exactly when the planes came from the host
//     (planes decoded by the GPU Huffman kernel arrive with a bound, see lep_huff.cu).
//
// Bit-exactness notes follow the oracle (oracle/lepton_oracle.c), which is pinned against the reference.
#include "lep_common.cuh"
#include "lep_predict.cuh"

namespace lepb200 {

constexpr int ENC_WARPS_PER_CTA = 4;
constexpr int QCAP = 2944;   // two blocks in flight; worst case decisions per block: 6 + 49*22 + 2*(3 + 7*22) + 22 = 1420

// Decision items.  Symbolisation does not write the binary decisions one by one: every coded coefficient leaves ONE
// 16-byte descriptor (exponent / sign / residual / threshold branch bases, magnitude, sign, first queue position) and
// one byte in `mark` at its first queue position; the flush expands positions to (branch index, bit) pairs 32 at a time.
//   coefficient: w0 = exp base | len << 20 | sign << 24          w1 = sign branch | |v| << 20
//                w2 = residual base | first position << 20       w3 = threshold base | min_threshold << 20 (15 = none)
//   single decision ("raw"): w0 = 1 << 31, w1 = (bit << 31) | branch
// Item ids are fixed: 0..5 7x7 count bits, 6..54 7x7 coefficients (zig-zag), 55..57 / 65..67 edge counts, 58..64 /
// 68..74 edge coefficients, 75 the DC.
constexpr int N_ITEMS = 76;
constexpr int IT_NZ = 0, IT_77 = 6, IT_HCNT = 55, IT_H = 58, IT_VCNT = 65, IT_V = 68, IT_DC = 75;

struct EncWarpSmem {
    uint4 desc[2 * N_ITEMS];  // items of block A (ids 0..99) and block B (100..199) of the pair in flight
    uint8_t mark[QCAP];       // item id + 1 at the first queue position of each item, 0 elsewhere (kept zero between flushes)
    // flat arrays addressed by integer offsets: per-lane SELECTED pointers into shared memory would be generic pointers
    // (window base from a special register at every use)
    int16_t rast[5 * 64];     // raster-order copies: three rotating buffers (A, B, left neighbour of A) + above A, above B
    int32_t tmp[2 * 64];      // IDCT intermediates of A and B
    int16_t pix[2 * 64];      // IDCT outputs (pixels sans DC) of A and B
    // per-component tables of the image, copied at every row start: the IDCT, the Lakhani predictors and the threshold
    // contexts read them per block, and as loads from the image descriptor in global memory they accounted for a tenth of
    // the kernel's stall samples
    int32_t icx[64], icy[64]; // model.hh:254-255
    uint16_t qtab[64];        // quantisation table, raster order
    uint8_t mthr[64];         // model.hh:277-289
};

// (the CTA's shared memory is declared as separate arrays inside the kernel: members of one struct reached through a
// reference made the compiler build generic addresses -- shared-window base from a special register -- at several uses)

// ---- queue flush: expansion of the items + batched model update ---------------------------------------
__device__ __forceinline__ uint32_t expand_item(const uint4 d, int pos) {      // pos: position relative to the item's block
    if (d.x >> 31) return d.y;
    const int len = (int)((d.x >> 20) & 15u), nexp = min(len + 1, 11);
    const int k = pos - (int)(d.z >> 20);
    if (k < nexp) return ((d.x & 0xfffffu) + (uint32_t)k) | ((uint32_t)(len != k) << 31);
    if (k == nexp) return (d.y & 0xfffffu) | (((d.x >> 24) & 1u) << 31);
    const int ib = len - 2 - (k - nexp - 1);                  // residual bit index, MSB first
    const uint32_t av = d.y >> 20;
    const uint32_t bit = (av >> ib) & 1u;
    // threshold-coded bits (edges): branch chosen by the bits already sent, i.e. the magnitude's prefix (model.hh:1085-1100)
    const uint32_t addr = ib >= (int)((d.w >> 20) & 15u) ? (d.w & 0xfffffu) + min(av >> (ib + 1), 127u) : (d.z & 0xfffffu) + (uint32_t)ib;
    return addr | (bit << 31);
}

// n queued positions; the items of block B (ids >= N_ITEMS) are positioned relative to base_b
__device__ __forceinline__ void flush_queue(EncWarpSmem& ws, int n, int base_b, uint16_t* __restrict__ model,
                                            const uint32_t* __restrict__ s_rcp, uint16_t* __restrict__ tokens, uint32_t& ntok,
                                            uint32_t tok_cap, int lane) {
    const uint32_t lt_mask = (1u << lane) - 1, le_mask = lt_mask | (1u << lane);
    uint32_t carry = 0;                                        // item covering the last position of the previous batch
    // decision (branch index, bit) of queue position `pos` for this lane; 0 past the end
    auto decision_at = [&](int pos) -> uint32_t {
        // which item covers the position: nearest start mark at or below it
        const uint32_t mk = ws.mark[pos];
        ws.mark[pos] = 0;
        const uint32_t starts = __ballot_sync(FULL, mk != 0) & le_mask;
        const uint32_t from_lane = __shfl_sync(FULL, mk, starts ? 31 - __clz(starts) : 0);
        const uint32_t item = starts ? from_lane : carry;
        carry = __shfl_sync(FULL, item, 31);
        return pos < n ? expand_item(ws.desc[item - 1], item > (uint32_t)N_ITEMS ? pos - base_b : pos) : 0u;
    };
    // software pipeline: the next batch is expanded and its model words are requested (L1 prefetch) before the current
    // batch is resolved, so the adaptive-count loads of a batch overlap the arithmetic of the one before
    uint32_t e_next = decision_at(lane);
    for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        const bool active = i < n;
        const uint32_t e = e_next;
        if (base + 32 < n) {
            e_next = decision_at(i + 32);
#ifndef LEPB200_EMU      // (the CPU warp emulator of tests/emu has no use for a prefetch)
            if (i + 32 < n) asm volatile("prefetch.global.L1 [%0];" ::"l"(model + (e_next & 0xfffffu)));
#endif
        }
        const uint32_t addr = e & 0xfffffu, bit = e >> 31;
        const uint32_t peers = __match_any_sync(FULL, active ? addr : (0x100000u + lane));
        const uint32_t earlier = peers & lt_mask;
        uint32_t w = active ? (uint32_t)model[addr] : 0u;
        // Resolve same-branch conflicts in queue order.  While no count of the group can saturate inside this batch
        // (the common case) record_obs_and_update is a plain increment, so the state a lane sees is the loaded word
        // plus the number of zeros / ones its predecessors on the same branch observed: closed form, no rounds.
        const uint32_t ones = __ballot_sync(FULL, bit != 0);
        const uint32_t n1_all = __popc(peers & ones), n0_all = __popc(peers & ~ones);
        const bool plain = !active || ((w & 0xff) + n0_all <= 254u && (w >> 8) + n1_all <= 254u);   // low byte 0xff (special state) never passes
        // the two absorbing states: (255,1) seeing only zeros and the "neverseen" (1,255) seeing only ones do not move
        // (branch.hh:87-99); branches that always code the same bit sit there for good
        const bool stuck = (w == 0x00feu && n1_all == 0) || ((w & 0xff) == 0xffu && n0_all == 0);
        uint32_t neww;                                            // state after this lane's own observation
        if (__all_sync(FULL, plain || stuck)) {
            if (!stuck) w += __popc(earlier & ~ones) + (__popc(earlier & ones) << 8);
            neww = stuck ? w : w + (bit ? 0x100u : 1u);
        } else {
            // general path: in round r the lanes of rank r take over the state their predecessor (rank r-1, already
            // resolved) leaves behind after its own update.
            const int rank = __popc(earlier);
            const int pred = earlier ? 31 - __clz(earlier) : lane;     // previous decision on the same branch
            const int maxrank = __reduce_max_sync(FULL, rank);
            for (int r = 1; r <= maxrank; ++r) {
                const uint32_t after = branch_update(w, bit);
                const uint32_t from_pred = __shfl_sync(FULL, after, pred);
                if (rank == r) w = from_pred;
            }
            neww = branch_update(w, bit);
        }
        const uint32_t pb = branch_prob(w, s_rcp) | (bit << 8);
        if (active && (peers >> lane) == 1u) model[addr] = (uint16_t)neww;                    // last decision of its branch
        if (active && ntok + i < tok_cap) LEP_ST_STREAM(tokens, ntok + i, (uint16_t)pb);                    // coalesced 2-byte stores
        __syncwarp();                                                                         // order this batch's model stores before the next batch's loads
    }
    ntok += (uint32_t)n;
    __syncwarp();
}

// ---- helpers for symbolisation ------------------------------------------------------------------------
// number of queue entries for one coefficient coded with (exponent unary, sign, len-1 residual bits)
__device__ __forceinline__ int coef_entries(int len) { return len == 0 ? 1 : min(len + 1, 11) + len; }

// ---- two blocks per warp: lanes 0..15 serve block A (x), lanes 16..31 block B (x + 1) in the lane-sparse sections ----
// Lane-parallel 8x8 IDCT (DC forced to zero) of A on lanes 0..7 and of B on lanes 8..15.
__device__ __forceinline__ void warp_idct_pair(EncWarpSmem& ws, int offA, int offB, const uint16_t* __restrict__ q, int lane, bool has_b) {
    const int b = (lane >> 3) & 1, r = lane & 7;
    const bool act = lane < (has_b ? 16 : 8);
    if (act) {
        const int ro = b ? offB : offA;
        int32_t in[8], out[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) in[k] = (int32_t)ws.rast[ro + r * 8 + k] * (int32_t)q[r * 8 + k];
        if (r == 0) in[0] = 0;
        idct_row(in, out);
#pragma unroll
        for (int k = 0; k < 8; ++k) ws.tmp[b * 64 + r * 8 + k] = out[k];
    }
    __syncwarp();
    if (act) {
        int32_t in[8], out[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) in[k] = ws.tmp[b * 64 + k * 8 + r];
        idct_col(in, out);
#pragma unroll
        for (int k = 0; k < 8; ++k) ws.pix[b * 64 + k * 8 + r] = (int16_t)out[k];
    }
    __syncwarp();
}

// adv_predict_dc_pix for both halves at once (see warp_predict_dc): within a half, lanes 0..7 hold the left estimate,
// lanes 8..15 the above one.  po = offset of the half's pixels; has_left is per half; the result is uniform within a half.
__device__ __forceinline__ DcPred warp_predict_dc_pair(const EncWarpSmem& ws, int po, int left_v, int above_h, bool has_left, bool has_above, int q0, int lane) {
    int est = 0;
    const int i = lane & 7, hb = lane & 16;
    if ((lane & 8) == 0) {
        if (has_left) {
            int16_t p0 = ws.pix[po + i * 8], p1 = ws.pix[po + i * 8 + 1];
            int16_t delta = (int16_t)(p0 - p1);
            est = (int16_t)((int16_t)((int16_t)left_v - half_rz16(delta)) - (int16_t)(p0 + 1024));
        }
    } else {
        if (has_above) {
            int16_t p0 = ws.pix[po + i], p1 = ws.pix[po + 8 + i];
            int16_t delta = (int16_t)(p0 - p1);
            est = (int16_t)((int16_t)((int16_t)above_h - half_rz16(delta)) - (int16_t)(p0 + 1024));
        }
    }
    int s = grp8_sum(est), mn = grp8_min(est), mx = grp8_max(est);
    int sl = __shfl_sync(FULL, s, hb), sa = __shfl_sync(FULL, s, hb + 8);
    int mnl = __shfl_sync(FULL, mn, hb), mna = __shfl_sync(FULL, mn, hb + 8);
    int mxl = __shfl_sync(FULL, mx, hb), mxa = __shfl_sync(FULL, mx, hb + 8);
    DcPred r; r.pred = 0; r.unc = 0; r.unc2 = 0;
    int avgmed = 0;
    if (has_left || has_above) {
        int a0, a1, mn_all, mx_all;
        if (has_left && has_above) { a0 = sl; a1 = sa; mn_all = min(mnl, mna); mx_all = max(mxl, mxa); }
        else if (has_left) { a0 = a1 = sl; mn_all = mnl; mx_all = mxl; }
        else { a0 = a1 = sa; mn_all = mna; mx_all = mxa; }
        avgmed = (a0 + a1) >> 1;
        r.unc = (mx_all - mn_all) >> 3;
        a0 -= avgmed; a1 -= avgmed;
        int far_afield = a1;
        if (iabs(a0) < iabs(a1)) far_afield = a0;
        r.unc2 = far_afield >> 3;
    }
    r.pred = (div_trunc_small(avgmed, q0) + 4) >> 3;            // |avgmed| < 2^20
    return r;
}

// NeighborSummary::set_horizontal / set_vertical on the half's pixels (see edge_pixel): l < 8 right column, else bottom row
__device__ __forceinline__ int edge_pixel_at(const EncWarpSmem& ws, int po, int q0, int dc, int l) {
    const int i = l & 7;
    int16_t cur, prev;
    if (l < 8) { cur = ws.pix[po + i * 8 + 7]; prev = ws.pix[po + i * 8 + 6]; }
    else { cur = ws.pix[po + 56 + i]; prev = ws.pix[po + 48 + i]; }
    const int16_t delta = (int16_t)(cur - prev);
    const int16_t qdc = (int16_t)((uint32_t)q0 * (uint32_t)dc);
    return (int16_t)(cur + half_rz16(delta) + 1024 + qdc);
}

// compute_lak (see lak_pred) with the blocks given as offsets into the raster buffers
__device__ __forceinline__ int lak_pred_at(const EncWarpSmem& ws, int cur_off, int nb_off, const int32_t* __restrict__ icos, int first, int step) {
    uint32_t pred = (uint32_t)(int32_t)ws.rast[nb_off + first] * (uint32_t)icos[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) {
        const int32_t nbv = ws.rast[nb_off + first + i * step];
        const int32_t t = (int32_t)ws.rast[cur_off + first + i * step] + ((i & 1) ? nbv : -nbv);
        pred -= (uint32_t)icos[i] * (uint32_t)t;
    }
    const int32_t p = (int32_t)pred;
    const int32_t t = (p + ((p >> 31) & 8191)) >> 13;
    return div_trunc_small(t, icos[0] >> 13);
}

// ---- the kernel ---------------------------------------------------------------------------------------
#ifndef LEPB200_ENC_MINBLOCKS
#define LEPB200_ENC_MINBLOCKS 6
#endif
__global__ void __launch_bounds__(ENC_WARPS_PER_CTA * 32, LEPB200_ENC_MINBLOCKS)
lep_encode_kernel(const ImageDesc* __restrict__ images, SegDesc* __restrict__ segs, int nseg, const int* __restrict__ order,
                  int* __restrict__ work_counter, uint16_t* __restrict__ model_pool, uint8_t* __restrict__ row_pool,
                  size_t row_pool_stride, uint16_t* __restrict__ token_base) {
    __shared__ uint32_t s_rcp[512];
    __shared__ uint8_t s_a2r[64];          // aligned -> raster and nz -> bin tables: per-lane indices, so not in constant memory
    __shared__ uint8_t s_nzbin[64];
    __shared__ EncWarpSmem s_w[ENC_WARPS_PER_CTA];
    // read the special registers once: left to itself the compiler re-reads %tid.x / %laneid (S2R, slow) all over the
    // block loop instead of keeping two registers
    int lane, warp_in_cta;
    {
        unsigned l, t;
#ifndef LEPB200_EMU
        asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
        asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
#else                    // CPU warp emulator (tests/emu)
        t = threadIdx.x; l = t & 31u;
#endif
        lane = (int)l; warp_in_cta = (int)(t >> 5);
    }
    const int gwarp = blockIdx.x * ENC_WARPS_PER_CTA + warp_in_cta;
    for (int i = threadIdx.x; i < 512; i += blockDim.x) s_rcp[i] = i < 2 ? 0u : (uint32_t)((0x100000000ull + i - 1) / i);
    for (int i = threadIdx.x; i < 64; i += blockDim.x) { s_a2r[i] = c_aligned_to_raster[i]; s_nzbin[i] = i < 50 ? c_nonzero_to_bin[i] : 0; }
    __syncthreads();
    const int r0 = s_a2r[2 * lane], r1 = s_a2r[2 * lane + 1];      // raster positions of this lane's two coefficients
    EncWarpSmem& ws = s_w[warp_in_cta];
    uint16_t* model = model_pool + (size_t)gwarp * M_TOTAL;
    uint8_t* rowbuf = row_pool + (size_t)gwarp * row_pool_stride;
    const uint32_t lt_mask = (1u << lane) - 1;

    for (;;) {
        int job = 0;
        if (lane == 0) job = atomicAdd(work_counter, 1);
        job = __shfl_sync(FULL, job, 0);
        if (job >= nseg) break;
        const int sidx = order[job];
        SegDesc& sd = segs[sidx];
        const ImageDesc& g = images[sd.image];
        if (sd.status != ST_OK) continue;          // rejected on the host (e.g. zero quantiser, model.hh:257-262)

        // reset the model to the identity prior: zero fill (16-byte stores, coalesced)
        {
            uint4* m4 = reinterpret_cast<uint4*>(model);
            const uint4 z = make_uint4(0, 0, 0, 0);
            for (uint32_t i = lane; i < M_TOTAL / 8; i += 32) LEP_ST_STREAM(m4, i, z);
            uint32_t* mk4 = reinterpret_cast<uint32_t*>(ws.mark);        // the flush leaves the marks zero; a segment that ended on an error does not
            for (int i = lane; i < QCAP / 4; i += 32) mk4[i] = 0u;
        }
        __syncwarp();

        uint16_t* tokens = token_base + sd.tokens;               // sd.tokens = offset (in tokens) assigned by the pre-pass
        const uint32_t tok_cap = sd.tok_cap;
        uint32_t ntok = 0;

        // per-component row buffers: bottom-edge prediction (8 x int16) and 7x7 nonzero count of the row above
        // (offsets kept as scalars: arrays indexed by the component would live in local memory)
        const int bw0 = g.bch[0], bw1 = g.ncmp > 1 ? g.bch[1] : 0, bw2 = g.ncmp > 2 ? g.bch[2] : 0;
        const size_t nz_base = (size_t)(bw0 + bw1 + bw2) * 16;
        const int nzs0 = (bw0 + 15) & ~15, nzs1 = (bw1 + 15) & ~15;

        int status = ST_OK;
        unsigned long long ndec = 0;
        uint32_t top_mask = 7u;                 // bit c set: no row of component c coded yet in this segment
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
            const uint32_t* plane = reinterpret_cast<const uint32_t*>(g.plane[c]);
            const uint32_t* rowp = plane + (size_t)y * w * 32;
            const uint32_t* abovep = rowp - (size_t)w * 32;
            {
                const uint32_t* gq = reinterpret_cast<const uint32_t*>(g.q[c]);
                const uint32_t* gm = reinterpret_cast<const uint32_t*>(g.min_thr[c]);
                __syncwarp();
                reinterpret_cast<uint32_t*>(ws.qtab)[lane] = gq[lane];
                if (lane < 16) reinterpret_cast<uint32_t*>(ws.mthr)[lane] = gm[lane];
                ws.icx[lane] = g.icos_x[c][lane]; ws.icx[32 + lane] = g.icos_x[c][32 + lane];
                ws.icy[lane] = g.icos_y[c][lane]; ws.icy[32 + lane] = g.icos_y[c][32 + lane];
                __syncwarp();
            }
            const uint16_t* q = ws.qtab;
            const int q0 = q[0];
            int16_t* redge = reinterpret_cast<int16_t*>(rowbuf + (size_t)(c == 0 ? 0 : (c == 1 ? bw0 : bw0 + bw1)) * 16);
            uint8_t* rnz = rowbuf + nz_base + (c == 0 ? 0 : (c == 1 ? nzs0 : nzs0 + nzs1));

            // ---- the row, two blocks (A = x, B = x + 1) per iteration
            const bool hiB = lane >= 16;                     // this lane serves block B in the packed sections
            const int l = lane & 15;
            const uint32_t trunc_bc = (uint32_t)g.trunc_bc[c];
            uint32_t curA = rowp[lane], curB = w > 1 ? rowp[32 + lane] : 0u;
            uint32_t abvA = has_above ? LEP_LD_LAST(abovep, lane) : 0u, abvB = (has_above && w > 1) ? LEP_LD_LAST(abovep, 32 + lane) : 0u;
            uint32_t left = 0, aleft = 0;                    // left / above-left neighbours of A
            int left_v = 0;                                  // lanes 0..7: right-column edge prediction of A's left neighbour
            int nz_left = 0;
            int ra = 0, rb = 1, rl = 2;                      // roles of the three rotating raster buffers
            for (int x = 0; x < w; x += 2) {
                // a block at or past the truncation bound is not coded unless it is the first of its row
                // (vp8_encoder.cc:110-113,133-135)
                const bool has_b = x + 1 < w && (uint32_t)((size_t)y * w + x + 1) < trunc_bc;
                const bool more = has_b && x + 2 < w && (uint32_t)((size_t)y * w + x + 2) < trunc_bc;
                // prefetch the next pair of this row and of the row above
                uint32_t ncurA = 0, ncurB = 0, nabvA = 0, nabvB = 0;
                if (x + 2 < w) { ncurA = rowp[(size_t)(x + 2) * 32 + lane]; if (has_above) nabvA = LEP_LD_LAST(abovep, (size_t)(x + 2) * 32 + lane); }
                if (x + 3 < w) { ncurB = rowp[(size_t)(x + 3) * 32 + lane]; if (has_above) nabvB = LEP_LD_LAST(abovep, (size_t)(x + 3) * 32 + lane); }
                // ---------------- raster copies for the gathers (IDCT, Lakhani edge predictor)
                ws.rast[ra * 64 + r0] = (int16_t)h_lo(curA); ws.rast[ra * 64 + r1] = (int16_t)h_hi(curA);
                ws.rast[3 * 64 + r0] = (int16_t)h_lo(abvA); ws.rast[3 * 64 + r1] = (int16_t)h_hi(abvA);
                if (has_b) {
                    ws.rast[rb * 64 + r0] = (int16_t)h_lo(curB); ws.rast[rb * 64 + r1] = (int16_t)h_hi(curB);
                    ws.rast[4 * 64 + r0] = (int16_t)h_lo(abvB); ws.rast[4 * 64 + r1] = (int16_t)h_hi(abvB);
                }
                __syncwarp();
                const bool act_h = !hiB || has_b;                           // this half has a block
                const bool has_left_h = hiB ? true : x > 0;
                const int rcur = (hiB ? rb : ra) * 64, rabove = (hiB ? 4 : 3) * 64, rleft = (hiB ? ra : rl) * 64;   // offsets into ws.rast

                // ---------------- number of non-zeros in the 7x7 areas (aligned_block.hh:132-148)
                const bool in0 = 2 * lane < 49, in1 = 2 * lane + 1 < 49;
                const uint32_t mA0 = __ballot_sync(FULL, in0 && h_lo(curA) != 0), mA1 = __ballot_sync(FULL, in1 && h_hi(curA) != 0);
                const uint32_t mB0 = __ballot_sync(FULL, has_b && in0 && h_lo(curB) != 0), mB1 = __ballot_sync(FULL, has_b && in1 && h_hi(curB) != 0);
                const int nzA = __popc(mA0) + __popc(mA1), nzB = __popc(mB0) + __popc(mB1);
                const int nz_h = hiB ? nzB : nzA;

                // ---------------- pixels, DC prediction (encoder.cc:293-364) and neighbour summaries (block_context.hh:44-78)
                warp_idct_pair(ws, ra * 64, rb * 64, q, lane, has_b);
                const int dcA = h_hi(__shfl_sync(FULL, curA, 24)), dcB = h_hi(__shfl_sync(FULL, curB, 24));     // aligned index 49
                const int dc_h = hiB ? dcB : dcA;
                const int pix_h = hiB ? 64 : 0;                                        // offset of this half's pixels in ws.pix
                const int edge = act_h ? edge_pixel_at(ws, pix_h, q0, dc_h, l) : 0;    // l < 8: right column, l >= 8: bottom row
                const int edge_from_a = __shfl_sync(FULL, edge, lane & 7);           // A's right column -> B's left neighbour
                const int left_v_h = hiB ? edge_from_a : left_v;
                int above_h = 0;
                if (has_above && act_h && l >= 8) above_h = redge[(size_t)(x + (hiB ? 1 : 0)) * 8 + (l - 8)];
                DcPred dp = warp_predict_dc_pair(ws, pix_h, left_v_h, above_h, has_left_h, has_above, q0, lane);
                int dc_len, dc_v;
                {
                    const int adv = adv_unpredict(dc_h, false, dp.pred);
                    if (act_h && dc_h != adv_unpredict((int)(int16_t)adv, true, dp.pred)) status = ST_COEF_RANGE;
                    dc_v = (int)(int16_t)adv;
                    // a residual that round-trips can still need more than 11 bits (adv_unpredict wraps only once, and a
                    // large prediction leaves it far outside +-1024): the reference refuses it too (encoder.cc:341-343)
                    if (act_h && bitlen(iabs(dc_v) & 0xffff) > 11) status = ST_COEF_RANGE;
                    dc_len = min(bitlen(iabs(dc_v) & 0xffff), 11);
                }
                const int n_dc = coef_entries(dc_len);

                // ---------------- 7x7 coefficients: which are coded and how many decisions each takes (encoder.cc:219-285)
                const int bA0 = __popc(mA0 & lt_mask) + __popc(mA1 & lt_mask), bA1 = bA0 + ((mA0 >> lane) & 1);
                const int bB0 = __popc(mB0 & lt_mask) + __popc(mB1 & lt_mask), bB1 = bB0 + ((mB0 >> lane) & 1);
                const bool cA0 = in0 && bA0 < nzA, cA1 = in1 && bA1 < nzA, cB0 = in0 && bB0 < nzB, cB1 = in1 && bB1 < nzB;
                const int lA0 = bitlen(iabs(h_lo(curA)) & 0xffff), lA1 = bitlen(iabs(h_hi(curA)) & 0xffff);
                const int lB0 = bitlen(iabs(h_lo(curB)) & 0xffff), lB1 = bitlen(iabs(h_hi(curB)) & 0xffff);
                if ((cA0 && lA0 > 11) || (cA1 && lA1 > 11) || (cB0 && lB0 > 11) || (cB1 && lB1 > 11)) status = ST_COEF_RANGE;
                const int nA0 = cA0 ? coef_entries(min(lA0, 11)) : 0, nA1 = cA1 ? coef_entries(min(lA1, 11)) : 0;
                const int nB0 = cB0 ? coef_entries(min(lB0, 11)) : 0, nB1 = cB1 ? coef_entries(min(lB1, 11)) : 0;
                int tot7;
                const int sc7 = warp_excl_scan((nA0 + nA1) | ((nB0 + nB1) << 16), lane, tot7);      // both blocks in one scan
                const int tot7A = tot7 & 0xffff, tot7B = tot7 >> 16;

                // ---------------- edges (encoder.cc:39-184): within a half, lanes 0..6 horizontal coefficient k = l + 1,
                // lanes 8..14 vertical k = l - 7; lane 7 carries the vertical count bits, lane 15 the horizontal ones
                const bool is_h = l < 7, is_v = l >= 8 && l < 15;
                const int ek = is_h ? l + 1 : l - 7;
                const int ecoord = is_h ? ek : 8 * ek;
                int ev = 0;
                if ((is_h || is_v) && act_h) ev = ws.rast[rcur + ecoord];
                const uint32_t nzmask = __ballot_sync(FULL, ev != 0);
                const uint32_t hm = (nzmask >> (lane & 16)) & 0x7f, vm = (nzmask >> ((lane & 16) + 8)) & 0x7f;
                const int ne_h = __popc(hm), ne_v = __popc(vm);
                int eprior = 0;
                if (act_h && ((is_h && has_above) || (is_v && has_left_h)))        // one pass for both edges of both blocks
                    eprior = lak_pred_at(ws, rcur, is_h ? rabove : rleft, (is_h ? ws.icx : ws.icy) + ek * 8, ecoord, is_h ? 8 : 1);
                const uint32_t lt16 = (1u << l) - 1;
                const int ne_rem = is_h ? ne_h - __popc(hm & lt16) : ne_v - __popc(vm & ((lt16 >> 8) & 0x7f));
                const bool ecoded = (is_h || is_v) && ne_rem > 0;
                const int eav = iabs(ev) & 0xffff;
                const int elen_raw = bitlen(eav);
                if (ecoded && elen_raw > 11) status = ST_COEF_RANGE;
                const int elen = min(elen_raw, 11);
                int ecnt = ecoded ? coef_entries(elen) : 0;
                if (l == 7) ecnt = 3;                                               // vertical count bits sit between the two edges
                int etot_all;
                const int esc_all = warp_excl_scan(ecnt, lane, etot_all);
                const int etotA = __shfl_sync(FULL, esc_all, 16);                  // exclusive prefix at lane 16 == total of half A
                const int esc = hiB ? esc_all - etotA : esc_all;
                const int etot_h = hiB ? etot_all - etotA : etotA;
                // eob of the 7x7 area per block (for the edge-count contexts)
                int eobx, eoby;
                {
                    const bool eA0 = (mA0 >> lane) & 1, eA1 = (mA1 >> lane) & 1, eB0 = (mB0 >> lane) & 1, eB1 = (mB1 >> lane) & 1;
                    int ax = 0, ay = 0, bx = 0, by = 0;
                    if (eA0) { ax = r0 & 7; ay = r0 >> 3; }
                    if (eA1) { ax = max(ax, r1 & 7); ay = max(ay, r1 >> 3); }
                    if (eB0) { bx = r0 & 7; by = r0 >> 3; }
                    if (eB1) { bx = max(bx, r1 & 7); by = max(by, r1 >> 3); }
                    const int packed = __reduce_max_sync(FULL, ax) | (__reduce_max_sync(FULL, ay) << 4) | (__reduce_max_sync(FULL, bx) << 8) | (__reduce_max_sync(FULL, by) << 12);
                    eobx = (packed >> (hiB ? 8 : 0)) & 15; eoby = (packed >> (hiB ? 12 : 4)) & 15;
                }

                // ---------------- queue layout: [6 count bits][7x7][3 h-count][h coefs][3 v-count][v coefs][DC] per block
                const int n_dcA = __shfl_sync(FULL, n_dc, 0), n_dcB = __shfl_sync(FULL, n_dc, 16);
                const int qnA = 6 + tot7A + 3 + etotA + n_dcA;
                const int qnB = has_b ? 6 + tot7B + 3 + (etot_all - etotA) + n_dcB : 0;
                const int base_b = qnA;
                const int base_h = hiB ? base_b : 0;                                // queue position of this half's block
                const int tot7_h = hiB ? tot7B : tot7A;
                const int it0 = hiB ? N_ITEMS : 0;                                  // item ids of this half's block

                // ---------------- items: count bits of the 7x7 area (context model.hh:463-485)
                {
                    const int nz_above = (has_above && act_h) ? (int)rnz[x + (hiB ? 1 : 0)] : 0;
                    const int nzl = hiB ? nzA : nz_left;
                    int ctx = 0;
                    if (has_above && !has_left_h) ctx = (nz_above + 1) / 2;
                    else if (has_left_h && !has_above) ctx = (nzl + 1) / 2;
                    else if (has_left_h && has_above) ctx = (nz_above + nzl + 2) / 4;
                    if (l < 6 && act_h) {
                        const int bin = s_nzbin[ctx];
                        const int idx = 5 - l;                                      // bit index, MSB first
                        ws.desc[it0 + IT_NZ + l] = make_uint4(0x80000000u, m_nz7(ci, bin, idx, nz_h >> (idx + 1)) | ((uint32_t)((nz_h >> idx) & 1) << 31), 0u, 0u);
                        ws.mark[base_h + l] = (uint8_t)(it0 + IT_NZ + l + 1);
                    }
                }
                // ---------------- items: 7x7 coefficients, block A then block B (all lanes, two coefficients each)
#pragma unroll
                for (int blk = 0; blk < 2; ++blk) {
                    if (blk == 1 && !has_b) break;
                    const uint32_t cur = blk ? curB : curA, lf = blk ? curA : left, ab = blk ? abvB : abvA, al = blk ? abvA : aleft;
                    const bool hl = blk ? true : x > 0;
                    const int nz = blk ? nzB : nzA;
                    int off = (blk ? base_b : 0) + 6 + (blk ? (sc7 >> 16) : (sc7 & 0xffff));
                    const int pr0 = aavrg16(h_lo(lf), h_lo(ab), h_lo(al), hl, has_above);
                    const int pr1 = aavrg16(h_hi(lf), h_hi(ab), h_hi(al), hl, has_above);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const bool coded = blk ? (h ? cB1 : cB0) : (h ? cA1 : cA0);
                        if (coded) {
                            const int zz = 2 * lane + h;
                            const int v = h ? h_hi(cur) : h_lo(cur), av = iabs(v);
                            const int len = min(blk ? (h ? lB1 : lB0) : (h ? lA1 : lA0), 11);
                            const int prior = h ? pr1 : pr0;
                            const int left_nz = nz - (blk ? (h ? bB1 : bB0) : (h ? bA1 : bA0));
                            const int bin = s_nzbin[left_nz];
                            const int bsr = bitlen((uint32_t)min(iabs(prior), 1023));
                            const int coord = h ? r1 : r0;
                            const int it = blk * N_ITEMS + IT_77 + zz;
                            ws.desc[it] = make_uint4(m_exp7(ci, bin, zz, bsr) | ((uint32_t)len << 20) | ((uint32_t)(v >= 0) << 24),
                                                     m_sign(ci, 0, 0) | ((uint32_t)(av & 0x7ff) << 20),
                                                     m_resn(ci, coord, bin) | ((uint32_t)(off - (blk ? base_b : 0)) << 20), 15u << 20);
                            ws.mark[off] = (uint8_t)(it + 1);
                            off += coef_entries(len);
                        }
                    }
                }
                // ---------------- items: edge counts and edge coefficients (both blocks at once)
                {
                    const int ebase = base_h + 6 + tot7_h;                          // first of the three h-count bits
                    if ((l == 15 || l == 7) && act_h) {
                        const bool vert = l == 7;
                        const int ne = vert ? ne_v : ne_h;
                        const int eob = vert ? eoby : eobx;
                        int o = vert ? ebase + 3 + esc : ebase;
                        const int it = it0 + (vert ? IT_VCNT : IT_HCNT);
                        for (int i = 2; i >= 0; --i) {
                            ws.desc[it + 2 - i] = make_uint4(0x80000000u, m_nze(vert, ci, eob, (nz_h + 3) / 7, i, ne >> (i + 1)) | ((uint32_t)((ne >> i) & 1) << 31), 0u, 0u);
                            ws.mark[o++] = (uint8_t)(it + 2 - i + 1);
                        }
                    }
                    if (ecoded) {
                        const int off = ebase + 3 + esc;
                        const int zig15 = is_h ? ek - 1 : 6 + ek;
                        const int bsr = bitlen((uint32_t)min(iabs(eprior), 1023));
                        const int p16 = (int)(int16_t)eprior;                           // sign_array_8: int16 truncation (model.hh:1116)
                        const int sctx = p16 == 0 ? 0 : (p16 > 0 ? 1 : 2);
                        const int min_thr = ws.mthr[ecoord];
                        uint32_t w3 = 15u << 20;
                        if (elen - 2 >= min_thr) {
                            const int ctx_abs = iabs(eprior) & 0xffff;                  // uint16_t ctx_abs (model.hh:1079)
                            w3 = m_thr(ci, min(ctx_abs >> min_thr, 255), min(elen - min_thr, 7)) | ((uint32_t)min_thr << 20);
                        }
                        const int it = it0 + (is_h ? IT_H : IT_V) + ek - 1;
                        ws.desc[it] = make_uint4(m_expx(ci, ne_rem, zig15, bsr) | ((uint32_t)elen << 20) | ((uint32_t)(ev >= 0) << 24),
                                                 m_sign(ci, sctx, bsr) | ((uint32_t)(eav & 0x7ff) << 20),
                                                 m_resn(ci, ecoord, ne_rem) | ((uint32_t)(off - base_h) << 20), w3);
                        ws.mark[off] = (uint8_t)(it + 1);
                    }
                    // ---------------- item: DC (exponent / sign / residual like a coefficient, own branches; model.hh:560-640)
                    if (l == 0 && act_h) {
                        const int off = ebase + 3 + etot_h;
                        const int lm = min(bitlen((uint32_t)iabs(dp.unc) & 0xffff), 11), lo = min(bitlen((uint32_t)iabs(dp.unc2) & 0xffff), 16);
                        const int sctx = dp.unc2 >= 0 ? (dp.unc2 == 0 ? 3 : 2) : 1;
                        ws.desc[it0 + IT_DC] = make_uint4(m_expdc(lm, lo) | ((uint32_t)dc_len << 20) | ((uint32_t)(dc_v >= 0) << 24),
                                                          m_sign(ci, 0, sctx) | ((uint32_t)(iabs(dc_v) & 0x7ff) << 20),
                                                          m_resdc(lm) | ((uint32_t)(off - base_h) << 20), 15u << 20);
                        ws.mark[off] = (uint8_t)(it0 + IT_DC + 1);
                    }
                }
                __syncwarp();
                // ---------------- neighbour summaries for the row below and the next pair
                if (act_h && l >= 8) redge[(size_t)(x + (hiB ? 1 : 0)) * 8 + (l - 8)] = (int16_t)edge;
                if (l == 0 && act_h) rnz[x + (hiB ? 1 : 0)] = (uint8_t)nz_h;
                left_v = __shfl_sync(FULL, edge, (has_b ? 16 : 0) + (lane & 7));       // lanes 0..7: right column of the last block coded
                nz_left = has_b ? nzB : nzA;

                // ---------------- code the queued decisions
                status = __reduce_max_sync(FULL, status);
                if (status != ST_OK) break;
                flush_queue(ws, qnA + qnB, base_b, model, s_rcp, tokens, ntok, tok_cap, lane);
                ndec += (unsigned long long)(qnA + qnB);
                if (!more) break;
                aleft = abvB; left = curB;
                curA = ncurA; curB = ncurB; abvA = nabvA; abvB = nabvB;
                { const int t = rl; rl = rb; rb = ra; ra = t; }
            }
            if (status != ST_OK) break;
        }
        if (status == ST_OK && ntok > tok_cap) status = ST_OUT_OVERFLOW;
        if (lane == 0) {
            sd.ntok = ntok;
            sd.len = 0;
            sd.status = status;
            sd.ndecisions_lo = (uint32_t)ndec;
            sd.ndecisions_hi = (uint32_t)(ndec >> 32);
        }
        __syncwarp();
    }
}

// ---- kernel B: the range coder, one thread per segment ------------------------------------------------
// vpx_start_encode / vpx_write / vpx_stop_encode (src/vp8/encoder/boolwriter.cc:17-35, boolwriter.hh:48-118)
// over the (probability, bit) tokens produced by kernel A.  Per-thread state; bytes go straight to the segment's
// stream, the carry walks back over already written 0xff bytes exactly like the reference.
// The coder state is kept as a 64-bit window `acc` over the not-yet-emitted low end of the code value and the count
// `U` of bits in it (the reference keeps 24+8 bits and emits a byte as soon as one is complete, boolwriter.hh:88-112;
// here up to four decisions are absorbed before complete bytes are peeled off, so the per-decision chain is
// split/select/normalise only).  A byte leaves through a small staging state -- the last byte not yet written plus a
// run of pending 0xff bytes -- so a carry (bit U of acc) normally needs no memory access: it increments the staged byte
// and turns the 0xff run into zeros.  The byte sequence is identical to the reference's walk-back over memory
// (boolwriter.hh:96-105); the rare carry into a staged 0xff falls back to exactly that walk.
struct RcState { unsigned long long acc; uint32_t range; int U; uint32_t mpos, cap; uint8_t* buf; int cache; uint32_t run; };

__device__ __forceinline__ void rc_store(RcState& w, uint32_t byte) {
#ifndef LEPB200_EMU
    if (w.mpos < w.cap) asm volatile("st.global.u8 [%0], %1;" ::"l"(w.buf + w.mpos), "r"(byte) : "memory");
#else                    // CPU warp emulator (tests/emu)
    if (w.mpos < w.cap) w.buf[w.mpos] = (uint8_t)byte;
#endif
    w.mpos++;
}
// rare path: pending 0xff run, a 0xff byte arriving, or a carry into a pending 0xff
__device__ __forceinline__ void rc_emit_slow(RcState& w, uint32_t b, bool carry) {
    if (carry) {
        if (w.cache == 0xff || w.cache < 0) {
            // bytes past the capacity were never stored: the walk starts inside the stream (the segment reports overflow
            // and is coded again into a larger buffer, so the bytes it changes here do not matter, only that it stays in bounds)
            long x = (long)min(w.mpos, w.cap) - 1;
            while (x >= 0 && w.buf[x] == 0xff) { w.buf[x] = 0; --x; }
            if (x >= 0) w.buf[x] += 1;
            if (w.cache == 0xff) w.cache = 0;
        } else {
            w.cache += 1;
        }
        if (w.run > 0) {                    // the 0xff run overflows to zeros; the last zero stays pending
            rc_store(w, (uint32_t)w.cache);
            for (uint32_t i = 1; i < w.run; ++i) rc_store(w, 0);
            w.cache = 0;
            w.run = 0;
        }
    }
    if (b == 0xff) { w.run++; return; }
    if (w.cache >= 0) rc_store(w, (uint32_t)w.cache);
    for (uint32_t i = 0; i < w.run; ++i) rc_store(w, 0xff);
    w.cache = (int)b;
    w.run = 0;
}
__device__ __forceinline__ void rc_emit(RcState& w, uint32_t b, bool carry) {
    const bool fast = w.run == 0 && b != 0xff && w.cache >= 0 && !(carry && w.cache == 0xff);
    if (fast) {
        rc_store(w, (uint32_t)w.cache + (carry ? 1u : 0u));
        w.cache = (int)b;
    } else {
        rc_emit_slow(w, b, carry);
    }
}
// peel complete bytes off the top of the window (a byte is complete once 32 bits are pending, boolwriter.hh:88)
__device__ __forceinline__ void rc_drain(RcState& w) {
    while (w.U >= 32) {
        const uint32_t top = (uint32_t)(w.acc >> (w.U - 8));          // 8 bits + the carry above them
        w.acc &= (1ull << (w.U - 8)) - 1;
        w.U -= 8;
        rc_emit(w, top & 0xff, (top >> 8) != 0);
    }
}
// vpx_write minus the byte emission: 4 of these fit between two drains (U <= 31 + 4*7 + carry bit < 64)
__device__ __forceinline__ void rc_put(RcState& w, uint32_t bit, uint32_t prob) {
    const uint32_t split = 1 + (((w.range - 1) * prob) >> 8);
    uint32_t range = bit ? w.range - split : split;
    w.acc += bit ? split : 0u;
    const int shift = __clz(range) - 24;
    w.range = range << shift;
    w.acc <<= shift;
    w.U += shift;
}

constexpr int RC_THREADS = 32;

__global__ void __launch_bounds__(RC_THREADS)
lep_rangecode_kernel(SegDesc* __restrict__ segs, int nseg, const int* __restrict__ order, const uint16_t* __restrict__ token_base) {
    const int t = blockIdx.x * RC_THREADS + threadIdx.x;
    if (t >= nseg) return;
    SegDesc& sd = segs[order[t]];
    if (sd.status != ST_OK) return;
    RcState w;
    w.acc = 0; w.range = 255; w.U = 8; w.mpos = 0; w.cap = sd.cap; w.buf = reinterpret_cast<uint8_t*>(sd.stream);
    w.cache = -1; w.run = 0;
    rc_put(w, 0, 128);                                               // vpx_start_encode marker bit (boolwriter.cc:17-24)
    const uint16_t* tok = token_base + sd.tokens;
    const uint4* tok4 = reinterpret_cast<const uint4*>(tok);
    const uint32_t ntok = sd.ntok;
    const uint32_t nfull = ntok / 8;
    // RC_DEPTH loads of 16 bytes in flight per thread (a register ring, 8 tokens each): one thread per segment leaves
    // few loads in flight per SM, and the token streams (2 bytes per decision) have to arrive at a large fraction of HBM bandwidth
    constexpr int RC_DEPTH = 10;
    uint4 q[RC_DEPTH];
#pragma unroll
    for (int j = 0; j < RC_DEPTH; ++j) q[j] = (uint32_t)j < nfull ? __ldg(tok4 + j) : make_uint4(0, 0, 0, 0);
    for (uint32_t base = 0; base < nfull; base += RC_DEPTH) {
#pragma unroll
        for (int j = 0; j < RC_DEPTH; ++j) {
            const uint32_t i = base + (uint32_t)j;
            if (i < nfull) {
                const uint4 cur = q[j];
                q[j] = i + RC_DEPTH < nfull ? __ldg(tok4 + i + RC_DEPTH) : make_uint4(0, 0, 0, 0);
                rc_drain(w);
                rc_put(w, (cur.x >> 8) & 1, cur.x & 0xff);
                rc_put(w, (cur.x >> 24) & 1, (cur.x >> 16) & 0xff);
                rc_put(w, (cur.y >> 8) & 1, cur.y & 0xff);
                rc_put(w, (cur.y >> 24) & 1, (cur.y >> 16) & 0xff);
                rc_drain(w);
                rc_put(w, (cur.z >> 8) & 1, cur.z & 0xff);
                rc_put(w, (cur.z >> 24) & 1, (cur.z >> 16) & 0xff);
                rc_put(w, (cur.w >> 8) & 1, cur.w & 0xff);
                rc_put(w, (cur.w >> 24) & 1, (cur.w >> 16) & 0xff);
            }
        }
    }
#pragma unroll 1
    for (uint32_t i = nfull * 8; i < ntok; ++i) { const uint32_t v = tok[i]; rc_drain(w); rc_put(w, (v >> 8) & 1, v & 0xff); }
#pragma unroll 1
    for (int i = 0; i < 32; ++i) { rc_drain(w); rc_put(w, 0, 128); }   // vpx_stop_encode (boolwriter.cc:26-35)
    rc_drain(w);
    // drain the staging, then the trailing-marker rule of vpx_stop_encode (boolwriter.cc:32-34)
    uint32_t last = 0;
    if (w.cache >= 0) { rc_store(w, (uint32_t)w.cache); last = (uint32_t)w.cache; }
    for (uint32_t i = 0; i < w.run; ++i) { rc_store(w, 0xff); last = 0xff; }
    if (w.mpos > 0 && (last & 0xe0) == 0xc0) rc_store(w, 0);
    sd.len = w.mpos;
    if (w.mpos >= w.cap) sd.status = ST_OUT_OVERFLOW;
}

// ---- kernel B, parallel form -----------------------------------------------------------------------------
// The serial kernel above is a floor whatever the batch size: one dependent chain of every token of a segment on one thread.
// Two facts break the chain up (boolwriter.hh:48-118 read as arithmetic):
//   * `range` and the number of bits shifted out depend only on the (probability, bit) sequence, never on `lowvalue`;
//   * `lowvalue` is a plain sum: a 1-decision adds its `split` at the current bit position, and the byte stream is that
//     sum written out from the top (the carry walk of boolwriter.hh:96-105 is the carry of this addition).
// So: (1) lep_rangepass_kernel, still one thread per segment but with the short chain split -> select -> normalise only
// (no window, no bytes), records (range, bits shifted so far) every RC_PIECE tokens and the total; (2)
// lep_rangepiece_kernel gives every piece of RC_PIECE tokens to its own thread, which replays the range evolution from
// its checkpoint and ADDS its splits -- as 16-bit digits with room for deferred carries -- into the segment's digit array
// (pieces overlap by a digit or two at their borders: atomic adds); (3) lep_rangenorm_kernel resolves the carries from
// the last digit to the first and writes the bytes, the stop rule of vpx_stop_encode (boolwriter.cc:32-34) included.
// Depth of a bit = its distance from the top of the code value: the coder starts with an 8-bit window (depths 1..8); a
// split added after S shifted bits covers depths S+1..S+8; byte k of the stream is depths 8k+1..8k+8, digit d the bytes
// 2d, 2d+1; of the 8+T bits the last 24..31 never leave the window (vpx_stop_encode pushes 32 zero decisions through).
constexpr int RC_PIECE = 1024;

struct RcRange { uint32_t range; uint32_t S; };
__device__ __forceinline__ void rr_put(RcRange& r, uint32_t bit, uint32_t prob, uint32_t& split_out, int& shift_out) {
    const uint32_t split = 1 + (((r.range - 1) * prob) >> 8);
    const uint32_t range = bit ? r.range - split : split;
    const int shift = __clz(range) - 24;
    r.range = range << shift;
    r.S += (uint32_t)shift;
    split_out = split; shift_out = shift;
}

// (1) range-only pass: checkpoints ck[(tokens >> 10) + 2 * segment + piece] = S << 8 | range, total shift per segment.
// Still one thread per segment, so what counts is the dependent chain per token.  split -> select -> count leading
// zeros -> shift is seven dependent instructions; but a normalised
// range has only 128 values and a token 512, so the whole transition fits a 128 KB table in shared memory:
// entry[token * 128 + (range - 128)] = (new range - 128) << 1 | shift << 8, and the chain per token is one LOP3 (next byte
// offset = token row | state) and one 16-bit shared-memory load.  One CTA of 128 threads per SM holds the table.
constexpr int RCT_THREADS = 128;
constexpr int RCT_ENTRIES = 512 * 128;
constexpr int RCT_RING = 32;                                   // 16-byte token slots per thread in flight (power of two)
constexpr size_t RCT_SMEM_TABLE_BYTES = (size_t)RCT_ENTRIES * 2;
constexpr size_t RCT_SMEM_BYTES = RCT_SMEM_TABLE_BYTES + (size_t)RCT_RING * RCT_THREADS * 16;      // 128 KB table + 64 KB ring
// asynchronous 16-byte copy global -> shared (LDGSTS), commit / wait of the per-thread copy groups
__device__ __forceinline__ void rct_async16(uint4* dst_shared, const uint4* src_global) {
#ifndef LEPB200_EMU
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst_shared);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(d), "l"(src_global) : "memory");
#else
    *dst_shared = *src_global;
#endif
}
__device__ __forceinline__ void rct_commit() {
#ifndef LEPB200_EMU
    asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
__device__ __forceinline__ void rct_wait_ring() {               // at most RCT_RING - 1 groups still pending: the oldest slot has arrived
#ifndef LEPB200_EMU
    asm volatile("cp.async.wait_group %0;" :: "n"(RCT_RING - 1) : "memory");
#endif
}
__device__ __forceinline__ uint32_t rct_entry(uint32_t tok9, uint32_t range) {
    const uint32_t prob = tok9 & 0xff, bit = tok9 >> 8;
    const uint32_t split = 1 + (((range - 1) * prob) >> 8);
    uint32_t r = bit ? range - split : split;
    if (r == 0) return 0;                                   // probability 0 with bit 1: never produced by kernel A
    const int shift = __clz(r) - 24;
    r <<= shift;
    return ((r - 128) << 1) | ((uint32_t)shift << 8);
}
template <bool kAsyncFeed>
__global__ void __launch_bounds__(RCT_THREADS, 1)
lep_rangepass_kernel(SegDesc* __restrict__ segs, int nseg, const int* __restrict__ order, const uint16_t* __restrict__ token_base,
                     unsigned long long* __restrict__ ck) {
#ifndef LEPB200_EMU
    extern __shared__ uint16_t s_rct[];
#else
    static uint16_t s_rct[RCT_SMEM_BYTES / 2];
#endif
    for (int e = threadIdx.x; e < RCT_ENTRIES; e += RCT_THREADS) s_rct[e] = (uint16_t)rct_entry((uint32_t)e >> 7, 128u + ((uint32_t)e & 127u));
    __syncthreads();
    const int t = blockIdx.x * RCT_THREADS + threadIdx.x;
    if (t >= nseg) return;
    const int sidx = order[t];
    SegDesc& sd = segs[sidx];
    if (sd.status != ST_OK) { sd.total_shift = 0; return; }
    unsigned long long* myck = ck + (sd.tokens >> 10) + 2ull * (unsigned long long)sidx;
    const unsigned char* tab = reinterpret_cast<const unsigned char*>(s_rct);
    uint32_t e = (255u - 128u) << 1;                        // last entry read; e & 0xfe = (range - 128) << 1 = byte offset inside a token's row
    uint32_t S = 0;
    // one transition: address = row of the token (token << 8 bytes) | state, as ONE lop3 (the token row is ready long before)
#ifndef LEPB200_EMU
#define RCT_ADDR(dst, row) asm("lop3.b32 %0, %1, 0xfe, %2, 0xea;" : "=r"(dst) : "r"(e), "r"(row))      /* (e & 0xfe) | row */
#else
#define RCT_ADDR(dst, row) dst = (e & 0xfeu) | (row)
#endif
#define RCT_STEP(tok9) { const uint32_t row = (uint32_t)(tok9) << 8; uint32_t ad; RCT_ADDR(ad, row); e = *reinterpret_cast<const uint16_t*>(tab + ad); S += e >> 8; }
    myck[0] = 255ull;                                                   // piece 0 starts before the marker bit
    RCT_STEP(128u);                                                     // vpx_start_encode marker bit (boolwriter.cc:17-24)
    const uint16_t* tok = token_base + sd.tokens;
    const uint4* tok4 = reinterpret_cast<const uint4*>(tok);
    const uint32_t ntok = sd.ntok;
    const uint32_t nfull = ntok / 8;
    // Token feed: every thread streams its own tokens, 16 bytes (8 tokens) at a time.  With plain loads into a register
    // ring the kernel spent most of its stall samples waiting for tokens (a warp has six scoreboards, so of twelve loads in flight a wait also covers the younger load sharing the
    // scoreboard -- half the nominal distance).  The ring therefore lives in shared memory next to the table and is filled
    // with asynchronous copies (cp.async, LDGSTS: global -> shared without a register or a scoreboard in between):
    // RCT_RING slots of 16 bytes per thread, slot k of thread t at (k * RCT_THREADS + t) * 16 (a warp's 32 slots are 512
    // contiguous bytes), one commit group per slot, `cp.async.wait_group RCT_RING - 1` before a slot is read -- 256 tokens,
    // about 5 us of chain, between a request and its use.
    if (kAsyncFeed) {
        uint4* ring = reinterpret_cast<uint4*>(reinterpret_cast<unsigned char*>(s_rct) + RCT_SMEM_TABLE_BYTES) + threadIdx.x;
#pragma unroll 1
        for (uint32_t j = 0; j < (uint32_t)RCT_RING; ++j) { if (j < nfull) rct_async16(ring + j * RCT_THREADS, tok4 + j); rct_commit(); }
#pragma unroll 1
        for (uint32_t i = 0; i < nfull; ++i) {
            rct_wait_ring();
            uint4* slot = ring + (i & (uint32_t)(RCT_RING - 1)) * RCT_THREADS;
            const uint4 cur = *slot;
            if (i + RCT_RING < nfull) rct_async16(slot, tok4 + i + RCT_RING);
            rct_commit();
            if (i != 0 && (i & (RC_PIECE / 8 - 1)) == 0) myck[i / (RC_PIECE / 8)] = ((unsigned long long)S << 8) | (128u + ((e & 0xfeu) >> 1));
            RCT_STEP(cur.x & 0x1ffu); RCT_STEP((cur.x >> 16) & 0x1ffu);
            RCT_STEP(cur.y & 0x1ffu); RCT_STEP((cur.y >> 16) & 0x1ffu);
            RCT_STEP(cur.z & 0x1ffu); RCT_STEP((cur.z >> 16) & 0x1ffu);
            RCT_STEP(cur.w & 0x1ffu); RCT_STEP((cur.w >> 16) & 0x1ffu);
        }
    } else {
        // the round-2 feed before the ring (kept selectable for the A/B, LEPB200_RC_FEED=0): twelve plain 16-byte loads in
        // flight per thread in registers
        constexpr int RCT_DEPTH = 12;
        uint4 q[RCT_DEPTH];
#pragma unroll
        for (int j = 0; j < RCT_DEPTH; ++j) q[j] = (uint32_t)j < nfull ? __ldg(tok4 + j) : make_uint4(0, 0, 0, 0);
        for (uint32_t base = 0; base < nfull; base += RCT_DEPTH) {
#pragma unroll
            for (int j = 0; j < RCT_DEPTH; ++j) {
                const uint32_t i = base + (uint32_t)j;
                if (i < nfull) {
                    const uint4 cur = q[j];
                    q[j] = i + RCT_DEPTH < nfull ? __ldg(tok4 + i + RCT_DEPTH) : make_uint4(0, 0, 0, 0);
                    if (i != 0 && (i & (RC_PIECE / 8 - 1)) == 0) myck[i / (RC_PIECE / 8)] = ((unsigned long long)S << 8) | (128u + ((e & 0xfeu) >> 1));
                    RCT_STEP(cur.x & 0x1ffu); RCT_STEP((cur.x >> 16) & 0x1ffu);
                    RCT_STEP(cur.y & 0x1ffu); RCT_STEP((cur.y >> 16) & 0x1ffu);
                    RCT_STEP(cur.z & 0x1ffu); RCT_STEP((cur.z >> 16) & 0x1ffu);
                    RCT_STEP(cur.w & 0x1ffu); RCT_STEP((cur.w >> 16) & 0x1ffu);
                }
            }
        }
    }
#pragma unroll 1
    for (uint32_t i = nfull * 8; i < ntok; ++i) {
        if (i != 0 && (i & (RC_PIECE - 1)) == 0) myck[i / RC_PIECE] = ((unsigned long long)S << 8) | (128u + ((e & 0xfeu) >> 1));
        const uint32_t v = tok[i];
        RCT_STEP(v & 0x1ffu);
    }
#pragma unroll 1
    for (int i = 0; i < 32; ++i) RCT_STEP(128u);                        // vpx_stop_encode (boolwriter.cc:26-35)
#undef RCT_STEP
#undef RCT_ADDR
    sd.total_shift = S;
}

// Stream bytes of a segment that shifted T bits in all: L = (T - 16) >> 3 leave the window (boolwriter.hh:88), plus at most
// the one zero byte of the stop rule.  A segment whose L + 1 bytes may not fit below its capacity (the overflow check of
// lep_rangenorm_kernel is len >= cap) gets a slot of this size in the overflow arena instead.
__device__ __forceinline__ unsigned long long rc_overflow_bytes(const SegDesc& sd) {
    const unsigned long long T = sd.total_shift, L = T >= 16 ? (T - 16) >> 3 : 0;
    return L + 1 >= sd.cap ? (L + 2 + 255) & ~255ull : 0ull;
}

// exclusive scans of the digit counts -> digit offsets (total in *total_out), and of the overflow slots -> SegDesc::ovf (+
// the capacity of the slot; total in *ovf_total_out, 0 for every batch whose streams fit their capacity).  Without
// ovf_total_out the caller has no overflow arena: no stream moves, and one that does not fit reports ST_OUT_OVERFLOW.
// Single CTA (cf. lep_token_offsets_kernel).
__global__ void lep_digit_offsets_kernel(SegDesc* __restrict__ segs, int nseg, unsigned long long* __restrict__ total_out,
                                         unsigned long long* __restrict__ ovf_total_out = nullptr) {
    const bool grow = ovf_total_out != nullptr;
    __shared__ unsigned long long sums[1024], osums[1024];
    const int t = threadIdx.x, per = (nseg + 1023) / 1024;
    const int b = t * per, e = min(nseg, b + per);
    unsigned long long s = 0, o = 0;
    for (int i = b; i < e; ++i) { s += ((unsigned long long)segs[i].total_shift + 8 + 15) / 16 + 2; o += grow ? rc_overflow_bytes(segs[i]) : 0ull; }
    sums[t] = s;
    osums[t] = o;
    __syncthreads();
    if (t == 0) {
        unsigned long long run = 0, orun = 0;
        for (int i = 0; i < 1024; ++i) {
            unsigned long long v = sums[i], w = osums[i];
            sums[i] = run; run += v;
            osums[i] = orun; orun += w;
        }
        *total_out = run;
        if (grow) *ovf_total_out = orun;
    }
    __syncthreads();
    unsigned long long off = sums[t], ooff = osums[t];
    for (int i = b; i < e; ++i) {
        SegDesc& sd = segs[i];
        sd.digits = off; off += ((unsigned long long)sd.total_shift + 8 + 15) / 16 + 2;
        const unsigned long long ob = grow ? rc_overflow_bytes(sd) : 0ull;
        sd.ovf = ob ? ooff + 1 : 0;
        if (ob) { sd.cap = (uint32_t)ob; ooff += ob; }
    }
}

// (2) one thread per piece of RC_PIECE tokens: grid.y = segment, pieces strided over grid.x * blockDim.x threads.
// A thread carries five digits in registers: `top` = digit dn with room for carries, `win` = digits dn+1 .. dn+4 (bit 63 =
// depth 16 (dn + 1) + 1).  A split decided after S shifted bits lands with its bit 0 at depth S + 8 = bit `off` of win; when
// the position has moved on, the finished top digit leaves: with a plain store when no other piece can touch it (its 16
// depths lie strictly inside this piece's range), else with an atomic add.  The digits are checked every four tokens
// (<= 28 bits of movement), the same instruction for all lanes, so the lanes of a warp do not diverge per token.
constexpr int RCP_THREADS = 128;
struct RcDigits {
    uint32_t* dig; unsigned long long win; uint32_t top; int dn, off; uint32_t own_lo, own_hi;
    __device__ __forceinline__ void emit(int d, uint32_t v) {
        if (v == 0 || d < 0) return;
        const uint32_t first = 16u * (uint32_t)d + 1u;
        if (first > own_lo && first + 15u < own_hi) dig[d] = v; else atomicAdd(dig + d, v);
    }
    __device__ __forceinline__ void advance() {               // keeps off in [28, 44): room for four more tokens
        while (off < 28) { emit(dn, top); top = (uint32_t)(win >> 48); win <<= 16; ++dn; off += 16; }
    }
    __device__ __forceinline__ void flush() {
        emit(dn, top);
        emit(dn + 1, (uint32_t)(win >> 48)); emit(dn + 2, (uint32_t)(win >> 32) & 0xffffu);
        emit(dn + 3, (uint32_t)(win >> 16) & 0xffffu); emit(dn + 4, (uint32_t)win & 0xffffu);
    }
};
__global__ void __launch_bounds__(RCP_THREADS)
lep_rangepiece_kernel(const SegDesc* __restrict__ segs, int nseg, const uint16_t* __restrict__ token_base, const unsigned long long* __restrict__ ck,
                      uint32_t* __restrict__ digit_base) {
    const int sidx = blockIdx.y;
    if (sidx >= nseg) return;
    const SegDesc& sd = segs[sidx];
    if (sd.status != ST_OK) return;
    const uint32_t ntok = sd.ntok;
    const uint32_t npieces = max(1u, (ntok + RC_PIECE - 1) / RC_PIECE);
    const unsigned long long* myck = ck + (sd.tokens >> 10) + 2ull * (unsigned long long)sidx;
    const uint16_t* tok = token_base + sd.tokens;
    for (uint32_t p = blockIdx.x * RCP_THREADS + threadIdx.x; p < npieces; p += gridDim.x * RCP_THREADS) {
        const unsigned long long c = myck[p];
        RcRange r; r.range = (uint32_t)(c & 0xff); r.S = (uint32_t)(c >> 8);
        RcDigits g;
        g.dig = digit_base + sd.digits;
        g.win = 0; g.top = 0;
        g.dn = (int)((r.S + 36 + 15) / 16) - 5;
        g.off = 16 * (g.dn + 5) - (int)(r.S + 8);
        g.own_lo = r.S + 8;                                                // the previous piece reaches down to this depth
        g.own_hi = p + 1 < npieces ? (uint32_t)(myck[p + 1] >> 8) + 1 : 0xffffffffu;   // the next one starts here
        uint32_t sp; int sh;
        auto put = [&](uint32_t bit, uint32_t prob) {
            rr_put(r, bit, prob, sp, sh);
            if (bit) {
                const unsigned long long x = (unsigned long long)sp << g.off;
                g.win += x;
                g.top += g.win < x ? 1u : 0u;
            }
            g.off -= sh;
        };
        if (p == 0) { put(0, 128); g.advance(); }                          // marker bit
        const uint32_t t0 = p * RC_PIECE, t1 = min(ntok, t0 + RC_PIECE);
        uint32_t i = t0;
        for (; i + 8 <= t1; i += 8) {                                      // pieces start at multiples of 1024 tokens: 16-byte aligned
            const uint4 cur = __ldg(reinterpret_cast<const uint4*>(tok + i));
            put((cur.x >> 8) & 1, cur.x & 0xff); put((cur.x >> 24) & 1, (cur.x >> 16) & 0xff);
            put((cur.y >> 8) & 1, cur.y & 0xff); put((cur.y >> 24) & 1, (cur.y >> 16) & 0xff);
            g.advance();
            put((cur.z >> 8) & 1, cur.z & 0xff); put((cur.z >> 24) & 1, (cur.z >> 16) & 0xff);
            put((cur.w >> 8) & 1, cur.w & 0xff); put((cur.w >> 24) & 1, (cur.w >> 16) & 0xff);
            g.advance();
        }
        for (; i < t1; ++i) { const uint32_t v = tok[i]; put((v >> 8) & 1, v & 0xff); g.advance(); }
        if (p + 1 == npieces) for (int k = 0; k < 32; ++k) { put(0, 128); g.advance(); }   // stop bits: zeros, they only move the position
        g.flush();
    }
}

// (3) carries from the last digit to the first, bytes out; ONE WARP PER SEGMENT, 32 digits per step.
// A digit holds 16 bits plus whatever the pieces left above them.  Step one adds every digit's excess to its shallower
// neighbour; after that each digit owes at most one carry and the classical generate / propagate rule applies, which a
// warp resolves for 32 digits at once with two ballots and one 64-bit addition (bit j of (a + b + c) ^ a ^ b is the carry into
// position j when a = generate | propagate, b = generate).  Lane l holds digit base + l; carries run from lane 31 to lane 0.
constexpr int RCN_WARPS = 4;
__global__ void __launch_bounds__(RCN_WARPS * 32)
lep_rangenorm_kernel(SegDesc* __restrict__ segs, int nseg, const int* __restrict__ order, const uint32_t* __restrict__ digit_base,
                     uint8_t* __restrict__ ovf_base = nullptr) {
    const int t = blockIdx.x * RCN_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (t >= nseg) return;
    SegDesc& sd = segs[order[t]];
    if (sd.status != ST_OK) return;
    const uint32_t T = sd.total_shift;
    const uint32_t L = T >= 16 ? (T - 16) >> 3 : 0;                    // bytes that leave the window (boolwriter.hh:88)
    const uint32_t nd = (T + 8 + 15) / 16;
    const uint32_t* dig = digit_base + sd.digits;
    // a stream longer than its slot goes to the overflow arena (lep_digit_offsets_kernel sized the slot and set cap)
    uint8_t* buf = sd.ovf ? ovf_base + (sd.ovf - 1) : reinterpret_cast<uint8_t*>(sd.stream);
    const uint32_t cap = sd.cap;
    uint32_t g_prev = 0, c_prev = 0, last = 0;
    const int nbatch = (int)((nd + 31) / 32);
    uint32_t v_next = nbatch > 0 && (uint32_t)(nbatch - 1) * 32 + lane < nd ? dig[(uint32_t)(nbatch - 1) * 32 + lane] : 0u;
    for (int bt = nbatch - 1; bt >= 0; --bt) {
        const uint32_t d = (uint32_t)bt * 32 + (uint32_t)lane;
        const uint32_t v = v_next;
        if (bt > 0) v_next = dig[d - 32];                              // next step's digits are on their way while this one resolves
        const uint32_t r = v & 0xffffu, g = v >> 16;
        uint32_t g_in = __shfl_down_sync(FULL, g, 1);
        if (lane == 31) g_in = g_prev;
        const uint32_t u = r + g_in;
        const uint32_t r1 = u & 0xffffu;
        const uint32_t gm = __brev(__ballot_sync(FULL, (u >> 16) != 0)), pm = __brev(__ballot_sync(FULL, r1 == 0xffffu));
        const unsigned long long a = gm | pm, b = gm;
        const unsigned long long sum = a + b + c_prev;
        const uint32_t cin = (uint32_t)(sum ^ a ^ b);                  // bit 31 - lane: carry into this lane's digit
        const uint32_t fin = (r1 + ((cin >> (31 - lane)) & 1u)) & 0xffffu;
        c_prev = (uint32_t)(sum >> 32) & 1u;
        g_prev = __shfl_sync(FULL, g, 0);
        const uint32_t hi = fin >> 8, lo = fin & 0xffu, k = 2u * d;
        if (d < nd) {
            if (k + 1 < L && k + 1 < cap) *reinterpret_cast<uint16_t*>(buf + k) = (uint16_t)(hi | (lo << 8));
            else if (k < L && k < cap) buf[k] = (uint8_t)hi;
            if (L > 0 && k + 1 == L - 1) last = 0x100u | lo;
            if (L > 0 && k == L - 1) last = 0x100u | hi;
        }
    }
    last = __reduce_max_sync(FULL, last) & 0xffu;
    uint32_t len = L;
    if (L > 0 && (last & 0xe0) == 0xc0) { if (lane == 0 && len < cap) buf[len] = 0; ++len; }     // boolwriter.cc:32-34
    if (lane == 0) {
        sd.len = len;
        sd.stream = (unsigned long long)(uintptr_t)buf;               // where lep_compact_kernel and lep_gather_kernel find it
        if (len >= cap) sd.status = ST_OUT_OVERFLOW;
    }
}

// ---- pre-pass: upper bound of the number of tokens each segment will produce -------------------------------
// Exact for the 7x7 and edge coefficients (their decision counts depend only on the block itself), 22 for the DC
// (its value depends on the prediction), 12 for the three count fields.  One CTA per segment, one warp per block.
constexpr int CNT_THREADS = 256;

__global__ void __launch_bounds__(CNT_THREADS)
lep_count_kernel(const ImageDesc* __restrict__ images, SegDesc* __restrict__ segs, int nseg) {
    const int s = blockIdx.x;
    if (s >= nseg) return;
    SegDesc& sd = segs[s];
    const ImageDesc& g = images[sd.image];
    const int lane = lane_id(), wid = threadIdx.x >> 5, nw = CNT_THREADS / 32;
    const uint32_t lt_mask = (1u << lane) - 1;
    unsigned long long acc = 0;
    if (sd.status == ST_OK) {
        uint32_t index = 0;
        for (;;) {
            RowSpec rs = row_spec_from_index(index++, g);
            if (rs.done) break;
            if (rs.luma_y >= sd.max_y && !sd.is_last) break;
            if (rs.skip) continue;
            if (rs.luma_y < sd.min_y) continue;
            const int c = rs.component, w = g.bch[c];
            const uint32_t* rowp = reinterpret_cast<const uint32_t*>(g.plane[c]) + (size_t)rs.curr_y * w * 32;
            for (int x = wid; x < w; x += nw) {
                const uint32_t cur = rowp[(size_t)x * 32 + lane];
                const int v0 = h_lo(cur), v1 = h_hi(cur);
                const int l0 = min(bitlen((uint32_t)iabs(v0) & 0xffff), 11), l1 = min(bitlen((uint32_t)iabs(v1) & 0xffff), 11);
                // region of each half: 0 = 7x7 (idx < 49), 1 = DC (49), 2 = horizontal edge (50..56), 3 = vertical edge (57..63)
                const int i0 = 2 * lane, i1 = 2 * lane + 1;
                const int r0 = i0 < 49 ? 0 : (i0 == 49 ? 1 : (i0 < 57 ? 2 : 3)), r1 = i1 < 49 ? 0 : (i1 == 49 ? 1 : (i1 < 57 ? 2 : 3));
                int cnt = 0;
#pragma unroll
                for (int reg = 0; reg < 4; ++reg) {
                    if (reg == 1) continue;
                    const bool n0 = r0 == reg && v0 != 0, n1 = r1 == reg && v1 != 0;
                    const uint32_t m0 = __ballot_sync(FULL, n0), m1 = __ballot_sync(FULL, n1);
                    // a coefficient is coded while non-zeros remain at or after it (in index order within its region)
                    const bool later0 = ((m0 | m1) & ~lt_mask) != 0;                 // this lane or later lanes hold a non-zero
                    const bool later1 = (m1 >> lane) != 0 || ((m0 >> lane) >> 1) != 0;
                    if (r0 == reg && later0) cnt += coef_entries(l0);
                    if (r1 == reg && later1) cnt += coef_entries(l1);
                }
                cnt = __reduce_add_sync(FULL, cnt);
                if (lane == 0) acc += (unsigned long long)cnt + 12 + 22;
            }
        }
    }
    __shared__ unsigned long long part[CNT_THREADS / 32];
    if (lane == 0) part[wid] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int i = 0; i < nw; ++i) t += part[i];
        t = (t + 64 + 63) & ~63ull;                              // 128-byte aligned token streams
        sd.tok_cap = t > 0xffffff00ull ? 0xffffff00u : (uint32_t)t;
    }
}

// exclusive scan of tok_cap -> token stream offsets (in tokens); total in *total_out.  Single CTA.
__global__ void lep_token_offsets_kernel(SegDesc* __restrict__ segs, int nseg, unsigned long long* __restrict__ total_out) {
    __shared__ unsigned long long sums[1024];
    const int t = threadIdx.x, per = (nseg + 1023) / 1024;
    const int b = t * per, e = min(nseg, b + per);
    unsigned long long s = 0;
    for (int i = b; i < e; ++i) s += segs[i].tok_cap;
    sums[t] = s;
    __syncthreads();
    if (t == 0) {
        unsigned long long run = 0;
        for (int i = 0; i < 1024; ++i) { unsigned long long v = sums[i]; sums[i] = run; run += v; }
        *total_out = run;
    }
    __syncthreads();
    unsigned long long off = sums[t];
    for (int i = b; i < e; ++i) { segs[i].tokens = off; off += segs[i].tok_cap; }
}

}  // namespace lepb200
