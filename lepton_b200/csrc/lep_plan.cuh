// lep_plan.cuh -- host-side planning of the kernels' job descriptors, shared by the C ABI (lep_capi.cu) and the CPU warp
// emulator's harness (tests/emu/emu_kernels.cc); included after the kernel sources.
//
// No CUDA runtime calls: the functions fill caller-owned plans (so a context keeps their capacity between calls), and
// every address a plan holds is an offset into an arena.  The caller rebases: the library adds the device base of the
// arena, the emulator the base of a host vector.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/lepton_b200.h"
#include "lep_common.cuh"

namespace lepb200 {

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ------------------------------------------------------------------------------------------------ quantiser tables
// zig-zag position of each raster index (reference src/vp8/model/jpeg_meta.hh:13-23)
const uint8_t k_zigzag[64] = {
    0, 1, 5, 6, 14, 15, 27, 28, 2, 4, 7, 13, 16, 26, 29, 42, 3, 8, 12, 17, 25, 30, 41, 43, 9, 11, 18, 24, 31, 40, 44, 53,
    10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};
// first column of icos_base_8192_scaled (src/vp8/model/jpeg_meta.hh:48-58): entries [i*8]
const int k_icos_base_col0[8] = {8192, 11363, 10703, 9633, 8192, 6436, 4433, 2260};
// src/vp8/model/model.hh:264-274
const uint16_t k_freqmax[64] = {
    1024, 931, 985, 968, 1020, 968, 1020, 1020, 932, 858, 884, 840, 932, 838, 854, 854,
    985, 884, 871, 875, 985, 878, 871, 854, 967, 841, 876, 844, 967, 886, 870, 837,
    1020, 932, 985, 967, 1020, 969, 1020, 1020, 969, 838, 878, 886, 969, 838, 969, 838,
    1020, 854, 871, 870, 1010, 969, 1020, 1020, 1020, 854, 854, 838, 1020, 838, 1020, 838};

// ProbabilityTablesBase::set_quantization_table (src/vp8/model/model.hh:247-290).  A zero in the first row or column of
// the scaled IDCT is refused in both directions: on the decode side (filetype == LEPTON, model.hh:257) the reference
// goes on and would divide by zero.
inline int fill_quant(ImageDesc& d, int c, const uint16_t zz[64]) {
    uint16_t* q = d.q[c];
    for (int i = 0; i < 64; ++i) q[i] = zz[k_zigzag[i]];
    for (int r = 0; r < 8; ++r) {
        for (int i = 0; i < 8; ++i) {
            d.icos_x[c][r * 8 + i] = k_icos_base_col0[i] * (int)q[i * 8 + r];
            d.icos_y[c][r * 8 + i] = k_icos_base_col0[i] * (int)q[r * 8 + i];
        }
        if (d.icos_x[c][r * 8] == 0 || d.icos_y[c][r * 8] == 0) return LEPB200_ST_UNSUPPORTED_JPEG_WITH_ZERO_IDCT_0;
    }
    for (int k = 0; k < 64; ++k) {
        uint16_t fm = (uint16_t)(k_freqmax[k] + q[k] - 1);
        if (q[k]) fm = (uint16_t)(fm / q[k]);
        int len = 0;
        for (uint32_t v = fm; v; v >>= 1) ++len;
        d.min_thr[c][k] = (uint8_t)(len > 7 ? len - 7 : 0);
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------ coder batches
// Rows of component c coded by a segment [min_y, max_y) (row iteration of lepton_codec.hh:41-100).
inline size_t segment_blocks(const lepb200_image& im, int min_y, int max_y, bool last) {
    size_t n = 0;
    int v0 = im.bcv[0] / im.mcuv;
    for (int c = 0; c < im.ncmp; ++c) {
        int mult = im.bcv[c] / im.mcuv;
        long y0 = (long)(min_y / std::max(v0, 1)) * mult, y1 = last ? im.trunc_bcv[c] : (long)((max_y + v0 - 1) / std::max(v0, 1)) * mult;
        y1 = std::min<long>(y1, im.trunc_bcv[c]);
        if (y1 > y0) n += (size_t)(y1 - y0) * im.bch[c];
    }
    return n;
}

// nullptr, or what is wrong with the image descriptor
inline const char* validate_image(const lepb200_image& im) {
    if (im.ncmp < 1 || im.ncmp > 3 || im.mcuv <= 0 || im.nseg < 1 || im.nseg > LEPB200_MAX_SEGMENTS) return "invalid image descriptor (ncmp/mcuv/nseg)";
    for (int c = 0; c < im.ncmp; ++c) {
        if (im.bch[c] <= 0 || im.bcv[c] <= 0 || im.bcv[c] % im.mcuv || im.trunc_bcv[c] < 0 || im.trunc_bcv[c] > im.bcv[c] ||
            im.trunc_bc[c] < 0 || (long long)im.trunc_bc[c] > (long long)im.bch[c] * im.bcv[c] || !im.planes[c])
            return "invalid component geometry";
    }
    for (int s = 0; s + 1 < im.nseg; ++s)
        if (im.luma_y_start[s] > im.luma_y_start[s + 1]) return "segment starts must be non-decreasing";
    return nullptr;
}

// Token slot of a segment whose decisions are bounded by `bound`: 64 tokens of slack, rounded up to 64 (piece checkpoints
// of the parallel range coder sit at (tokens >> 10) + 2 * segment).
inline uint32_t token_slot(unsigned long long bound) {
    const unsigned long long tcap = (bound + 64 + 63) & ~63ull;
    return tcap > 0xffffff00ull ? 0xffffff00u : (uint32_t)tcap;
}

struct BatchPlan {
    std::vector<ImageDesc> images;        // plane[c]: offset in the plane arena
    std::vector<SegDesc> segs;            // stream: offset in the stream arena; tokens: offset in the token arena (tokens_known)
    std::vector<int> order;               // bool-coded segments, then rANS-coded ones, each part largest first
    int order_ans = 0;                    // order[order_ans ..] are the rANS-coded segments (CODER_ANS)
    // encode batches with rANS-coded segments: segs holds the bool-coded segments first, then the rANS-coded ones (each in
    // image order), so that the range coder's launches, which take segments by index, take only the first order_ans;
    // seg_out[d] = the caller's index (image after image) of segs[d].  Empty: segs is in the caller's order.
    std::vector<int> seg_out;
    std::vector<size_t> seg_blocks;       // blocks each segment codes
    std::vector<size_t> plane_bytes;      // per image * 3 + component
    size_t plane_total = 0, stream_total = 0, row_stride = 0;
    bool tokens_known = false;            // encode: every segment came with a caller-supplied bound (no counting pre-pass)
    unsigned long long token_total = 0;   // ... and the token arena they add up to
};

// Job tables of an encode (in = nullptr) or decode batch (in = one stream per segment): ImageDesc / SegDesc, the plane arena
// (256-byte aligned planes), the stream arena, the row stride of the kernels' row buffers and the launch order.  coders
// (optional): the entropy coder of each image's streams (LEPB200_CODER_BOOL / LEPB200_CODER_ANS); nullptr = all bool.
// Returns nullptr, or what is wrong with the batch.
inline const char* plan_batch(BatchPlan& b, const lepb200_image* images, int nimages, bool encode, const lepb200_stream* in,
                              const uint8_t* coders = nullptr) {
    if (nimages <= 0 || !images) return "empty batch";
    b.images.assign(nimages, ImageDesc());
    b.segs.clear(); b.seg_blocks.clear(); b.seg_out.clear(); b.plane_bytes.assign((size_t)nimages * 3, 0);
    b.plane_total = b.stream_total = b.row_stride = 0;
    b.token_total = 0;
    b.tokens_known = encode;
    int sidx = 0;
    for (int i = 0; i < nimages; ++i) {
        const lepb200_image& im = images[i];
        if (const char* e = validate_image(im)) return e;
        if (coders && coders[i] > LEPB200_CODER_ANS) return "invalid entropy coder";
        ImageDesc& d = b.images[i];
        memset(&d, 0, sizeof(d));
        d.ncmp = im.ncmp; d.mcuv = im.mcuv;
        d.coder = coders && coders[i] == LEPB200_CODER_ANS ? CODER_ANS : CODER_BOOL;
        int qstatus = 0;
        size_t rs = 0;
        for (int c = 0; c < im.ncmp; ++c) {
            d.bch[c] = im.bch[c]; d.bcv[c] = im.bcv[c]; d.trunc_bcv[c] = im.trunc_bcv[c]; d.trunc_bc[c] = im.trunc_bc[c];
            d.mult[c] = im.bcv[c] / im.mcuv;
            int qs = fill_quant(d, c, im.qtable_zigzag[c]);
            if (qs) qstatus = qs;
            size_t pb = (size_t)im.bch[c] * im.bcv[c] * 128;
            b.plane_bytes[(size_t)i * 3 + c] = pb;
            d.plane[c] = b.plane_total;
            b.plane_total += align_up(pb, 256);
            rs += (size_t)im.bch[c] * 16 + align_up((size_t)im.bch[c], 16);
        }
        b.row_stride = std::max(b.row_stride, align_up(rs, 256));
        for (int s = 0; s < im.nseg; ++s, ++sidx) {
            SegDesc sd;
            memset(&sd, 0, sizeof(sd));
            sd.image = i;
            sd.min_y = im.luma_y_start[s];
            sd.is_last = s + 1 == im.nseg;
            sd.max_y = sd.is_last ? im.bcv[0] : im.luma_y_start[s + 1];
            sd.status = qstatus;
            size_t nb = segment_blocks(im, sd.min_y, sd.max_y, sd.is_last);
            b.seg_blocks.push_back(nb);
            if (encode) {
                // 64 B/block is > 1.5x what q=100 photos need.  Dense noise needs more (up to about 7/8 byte per decision):
                // such a stream moves to the overflow arena, sized from the exact length (parallel range coder, see
                // lep_digit_offsets_kernel) or from a proven bound when the serial coder codes the segment again
                // (plan_serial_rerun).  No stream is ever cut short.
                // An rANS segment's stream is written into its token slot (lep_anspass_kernel): no stream slot.
                size_t cap = d.coder == CODER_ANS ? 0 : align_up(nb * 64 + 4096, 256);
                sd.stream = b.stream_total; sd.cap = (uint32_t)cap;
                b.stream_total += cap;
                sd.tokens = 0; sd.tok_cap = 0;                    // assigned on the device by the counting pre-pass ...
                if (im.seg_token_bound[s]) {                      // ... unless the caller knows a bound (GPU Huffman decoder)
                    sd.tok_cap = token_slot(im.seg_token_bound[s]);
                    sd.tokens = b.token_total;
                    b.token_total += sd.tok_cap;
                } else {
                    b.tokens_known = false;
                }
            } else {
                sd.stream = b.stream_total; sd.cap = (uint32_t)in[sidx].len;
                b.stream_total += align_up((size_t)in[sidx].len + 16, 16);
            }
            b.segs.push_back(sd);
        }
    }
    const int nseg = (int)b.segs.size();
    auto coder = [&](int x) { return b.images[b.segs[x].image].coder; };
    if (encode && std::any_of(b.images.begin(), b.images.end(), [](const ImageDesc& d) { return d.coder == CODER_ANS; })) {
        b.seg_out.resize(nseg);
        for (int i = 0; i < nseg; ++i) b.seg_out[i] = i;
        std::stable_partition(b.seg_out.begin(), b.seg_out.end(), [&](int x) { return coder(x) != CODER_ANS; });
        std::vector<SegDesc> segs(nseg);
        std::vector<size_t> blocks(nseg);
        for (int d = 0; d < nseg; ++d) { segs[d] = b.segs[b.seg_out[d]]; blocks[d] = b.seg_blocks[b.seg_out[d]]; }
        b.segs.swap(segs);
        b.seg_blocks.swap(blocks);
    }
    // largest segments first (longest-processing-time-first on the persistent warps); a kernel launch takes the segments
    // of one coder, so those of the rANS coder follow all the others
    b.order.resize(nseg);
    for (int i = 0; i < nseg; ++i) b.order[i] = i;
    std::stable_sort(b.order.begin(), b.order.end(), [&](int x, int y) {
        return coder(x) != coder(y) ? coder(x) < coder(y) : b.seg_blocks[x] > b.seg_blocks[y]; });
    b.order_ans = nseg;
    while (b.order_ans > 0 && coder(b.order[b.order_ans - 1]) == CODER_ANS) --b.order_ans;
    return nullptr;
}

// ------------------------------------------------------------------------------------------------ range coder
// Parallel range coder: checkpoints of the range-only pass (unsigned long long each) for a token arena of token_total.
inline size_t rc_checkpoints(unsigned long long token_total, int nseg) { return ((size_t)token_total >> 10) + 2 * (size_t)nseg + 8; }

// Serial range coder: it learns a stream's length only by writing it, so a stream longer than its slot comes back with
// ST_OUT_OVERFLOW (kernel A's token overflow, ntok > tok_cap, is the other source of that status and stays an error).  Its
// tokens are still in the arena: lep_rangecode_kernel codes those segments again, alone, into the overflow arena, with a
// capacity no stream can reach.  Bound: before every decision the range is normalised (>= 128), and the sub-range kept is
// >= 1 (split >= 1, and split <= 1 + (range - 1) * 255 / 256 < range), so a decision shifts at most 7 bits; with the
// marker bit and the 32 stop decisions a segment shifts T <= 7 (ntok + 33) bits, and writes at most (T - 16) / 8 bytes
// plus the zero byte of the stop rule.
inline size_t serial_stream_bound(uint32_t ntok) { return align_up((7ull * ((unsigned long long)ntok + 33) + 8) / 8 + 2, 256); }

// The segments (of the records hs, fetched after the serial coder) to code again, into `redo`; their records get a slot in
// the overflow arena (stream = offset) and are reset.  Returns the size of that arena (0: nothing to code again).
inline size_t plan_serial_rerun(SegDesc* hs, int nseg, std::vector<int>& redo) {
    redo.clear();
    size_t total = 0;
    for (int s = 0; s < nseg; ++s) {
        if (hs[s].status != ST_OUT_OVERFLOW || hs[s].ntok > hs[s].tok_cap) continue;
        redo.push_back(s);
        hs[s].stream = total;
        hs[s].cap = (uint32_t)serial_stream_bound(hs[s].ntok);
        hs[s].status = ST_OK; hs[s].len = 0;
        total += hs[s].cap;
    }
    return total;
}

// ------------------------------------------------------------------------------------------------ Huffman tables
// Device tables of the DHT tables of a batch, built once per distinct DHT (most files share the standard ones).  A table
// that failed to build fails every job that uses it.
template <class Table> struct TableSet {
    std::vector<Table> tabs;
    std::vector<const lepb200_hufftable*> src;     // the DHT input of each entry
    std::vector<char> built;
    void clear() { tabs.clear(); src.clear(); built.clear(); }
    template <class Build> int index(const lepb200_hufftable& t, bool& ok, Build build) {
        for (size_t q = 0; q < src.size(); ++q)
            if (!memcmp(src[q], &t, sizeof(t))) { if (!built[q]) ok = false; return (int)q; }
        Table e;
        const bool b = build(t, e);
        if (!b) ok = false;
        tabs.push_back(e);
        built.push_back(b ? 1 : 0);
        src.push_back(&t);
        return (int)tabs.size() - 1;
    }
};

// ------------------------------------------------------------------------------------------------ Huffman decode
struct HuffDecodePlan {
    std::vector<HuffJob> jobs;            // huff, rows, plane[c]: offsets in the scan, row and plane arenas
    TableSet<HuffTableDev> tabs;
    std::vector<uint32_t> sub_base;       // n + 1: first sub-sequence of each job (lep_huffpar.cu)
    size_t plane_total = 0, huff_total = 0, rows_total = 0;
    uint32_t sub_total = 0;
    bool in_place = false;                // the scans lie in the staging range: their offsets are where they lie
};

// Jobs of lep_huffdecode_kernel and, with `subseq`, of the sub-sequence kernels (sub_bits bits per sub-sequence) for n
// scans; placeholders (entropy = nullptr) get a plane slot and HUFF_JOB_SKIP.  stage / stage_cap: the pinned staging
// buffer the caller may have de-stuffed the scans into, 16-byte aligned with >= 16 spare bytes after each (nullptr: none);
// scans that lie there are decoded where they lie.  Returns nullptr, or what is wrong with the batch.
inline const char* plan_huffman_decode(HuffDecodePlan& p, const lepb200_jpeg_scan* scans, int n, bool subseq, int sub_bits,
                                       const uint8_t* stage, size_t stage_cap) {
    p.jobs.assign(n, HuffJob());
    p.tabs.clear();
    p.sub_base.assign((size_t)n + 1, 0);
    p.plane_total = p.huff_total = p.rows_total = 0;
    p.sub_total = 0;
    int inside = 0, placeholders = 0;
    for (int i = 0; i < n; ++i)
        if (scans[i].entropy == nullptr) ++placeholders;
        else if (stage && scans[i].entropy >= stage && scans[i].entropy + scans[i].nbytes + 16 <= stage + stage_cap) ++inside;
    if (inside != 0 && inside != n - placeholders) return "huffman_decode_to_device: scans partly inside the staging buffer";
    p.in_place = inside > 0;
    for (int i = 0; i < n; ++i)
        if (p.in_place && scans[i].entropy && ((scans[i].entropy - stage) & 15)) return "huffman_decode_to_device: staged scan not 16-byte aligned";
    auto build = [](const lepb200_hufftable& t, HuffTableDev& d) { return huff_build_table(t.bits, t.vals, d); };
    for (int i = 0; i < n; ++i) {
        const lepb200_jpeg_scan& sc = scans[i];
        HuffJob& jb = p.jobs[i];
        memset(&jb, 0, sizeof(jb));
        const bool placeholder = sc.entropy == nullptr;
        bool ok = sc.ncmp >= 1 && sc.ncmp <= 3 && sc.mcuh > 0 && sc.mcuv > 0 && (placeholder || sc.rows);
        jb.ncmp = sc.ncmp; jb.mcuh = sc.mcuh; jb.mcuv = sc.mcuv; jb.rsti = sc.rsti; jb.nbytes = sc.nbytes;
        for (int c = 0; ok && c < sc.ncmp; ++c) {
            jb.H[c] = sc.H[c]; jb.V[c] = sc.V[c];
            ok = ok && sc.H[c] >= 1 && sc.H[c] <= 2 && sc.V[c] >= 1 && sc.V[c] <= 2;
            jb.bch[c] = sc.mcuh * sc.H[c]; jb.bcv[c] = sc.mcuv * sc.V[c];
            jb.nch[c] = sc.nch[c]; jb.ncv[c] = sc.ncv[c];
            if (!placeholder) { jb.dc_tab[c] = p.tabs.index(sc.dc[c], ok, build); jb.ac_tab[c] = p.tabs.index(sc.ac[c], ok, build); }
            jb.plane[c] = p.plane_total;
            p.plane_total += align_up((size_t)jb.bch[c] * jb.bcv[c] * 128, 256);
        }
        jb.status = ok ? (placeholder ? HUFF_JOB_SKIP : 0) : LEPB200_ST_NOT_HANDLED;
        if (placeholder) {
            jb.huff = 0; jb.nbytes = 0;
        } else if (p.in_place) {
            jb.huff = (size_t)(sc.entropy - stage);
            p.huff_total = std::max(p.huff_total, align_up((size_t)jb.huff + sc.nbytes + 16, 16));
        } else {
            jb.huff = p.huff_total;
            p.huff_total += align_up((size_t)sc.nbytes + 16, 16);
        }
        jb.rows = p.rows_total;
        p.rows_total += (size_t)(sc.mcuv + 1) * sizeof(HuffRow);
        // interleaved scans without restart intervals and with enough data take the many-threads-per-image kernels
        const uint64_t bits = (uint64_t)sc.nbytes * 8;
        jb.sub_base = p.sub_total;
        if (subseq && jb.status == 0 && sc.ncmp > 1 && sc.rsti == 0 && bits >= 4ull * (uint64_t)sub_bits && bits < (1ull << 32))
            jb.nsub = (uint32_t)((bits + (uint64_t)sub_bits - 1) / (uint64_t)sub_bits);
        p.sub_total += jb.nsub;
        p.sub_base[i] = jb.sub_base;
    }
    p.sub_base[n] = p.sub_total;
    return nullptr;
}

// Hands the results back to the scans: done = the job records after the kernels, rows = the row arena as the host sees it,
// rows_base = its address in the jobs' `rows` fields.
inline void huffman_decode_results(lepb200_jpeg_scan* scans, int n, const HuffJob* done, const uint8_t* rows, unsigned long long rows_base) {
    static_assert(sizeof(HuffRow) == sizeof(lepb200_huffrow), "row record layout");
    for (int i = 0; i < n; ++i) {
        const HuffJob& jb = done[i];
        scans[i].status = jb.status == HUFF_JOB_SKIP ? 0 : jb.status;
        scans[i].padbit = jb.padbit;
        scans[i].end_bitpos = jb.end_bitpos;
        scans[i].nrows = jb.nrows;
        if (jb.nrows > 0) memcpy(scans[i].rows, rows + (jb.rows - rows_base), sizeof(HuffRow) * (size_t)std::min(jb.nrows, scans[i].mcuv + 1));
    }
}

// ------------------------------------------------------------------------------------------------ Huffman encode
// DHT as code/length per symbol (build_huffcodes, jpgcoder.cc:5508-5540)
inline bool build_enc_table(const lepb200_hufftable& in, HEncTable& t) {
    memset(&t, 0, sizeof(t));
    int code = 0, k = 0;
    for (int len = 1; len <= 16; ++len) {
        for (int i = 0; i < in.bits[len]; ++i, ++k, ++code) {
            if (k >= 256 || code >= (1 << len)) return false;        // over-subscribed table
            t.code[in.vals[k]] = (uint16_t)code;
            t.len[in.vals[k]] = (uint8_t)len;
        }
        if (code > (1 << len)) return false;
        code <<= 1;
    }
    return true;
}

struct HuffEncodePlan {
    std::vector<HEncImage> images;        // out: offset in the output arena
    std::vector<HEncSeg> segs;            // one per thread-segment, image after image
    TableSet<HEncTable> tabs;
    std::vector<size_t> off;              // per image: offset of its scan bytes in the output arena (SIZE_MAX = not encoded)
    std::vector<int> seg_first;           // per image: index of its first segment record
    std::vector<int> seg_count;           // per image: its number of segment records
    size_t total = 0;                     // bytes of the output arena
};

// Jobs of lep_huffencode_kernel for n images whose coefficient planes lie where geom[i].plane says (the decode batch's
// ImageDesc).  Images with scan_bytes = 0 are skipped; images the kernel cannot encode (sampling, tables, segment count)
// get status LEPB200_ST_NOT_HANDLED and scan_bytes = 0.  data / status of every image are reset.
inline void plan_huffman_encode(HuffEncodePlan& p, lepb200_henc_image* imgs, int n, const ImageDesc* geom) {
    p.images.assign(n, HEncImage());
    p.segs.clear();
    p.tabs.clear();
    p.off.assign(n, SIZE_MAX);
    p.seg_first.assign(n, -1);
    p.seg_count.assign(n, 0);
    p.total = 0;
    for (int i = 0; i < n; ++i) {
        lepb200_henc_image& im = imgs[i];
        im.data = nullptr; im.status = 0;
        HEncImage& d = p.images[i];
        memset(&d, 0, sizeof(d));
        if (im.scan_bytes == 0) continue;
        const ImageDesc& g = geom[i];
        bool ok = im.nseg >= 1 && im.nseg <= LEPB200_MAX_SEGMENTS && g.ncmp >= 1 && g.ncmp <= 3;
        d.ncmp = g.ncmp; d.mcuv = g.mcuv; d.rsti = im.rsti; d.padbit = im.padbit; d.scan_len = im.scan_bytes;
        for (int c = 0; ok && c < g.ncmp; ++c) {
            ok = im.H[c] >= 1 && im.H[c] <= 2 && im.V[c] >= 1 && im.V[c] <= 2 && g.bch[c] % im.H[c] == 0 && g.bcv[c] == g.mcuv * im.V[c];
            d.H[c] = im.H[c]; d.V[c] = im.V[c]; d.bch[c] = g.bch[c]; d.plane[c] = g.plane[c];
            if (ok) { d.dc_tab[c] = p.tabs.index(im.dc[c], ok, build_enc_table); d.ac_tab[c] = p.tabs.index(im.ac[c], ok, build_enc_table); }
        }
        if (ok) {
            d.mcuh = g.bch[0] / im.H[0];
            for (int c = 1; ok && c < g.ncmp; ++c) ok = g.bch[c] / im.H[c] == d.mcuh;
        }
        if (!ok) { im.status = LEPB200_ST_NOT_HANDLED; im.scan_bytes = 0; continue; }
        p.off[i] = p.total;
        d.out = p.total;
        p.seg_first[i] = (int)p.segs.size();
        p.seg_count[i] = im.nseg;
        uint32_t off = 0;
        for (int k = 0; k < im.nseg; ++k) {
            HEncSeg sg;
            memset(&sg, 0, sizeof(sg));
            sg.image = i; sg.my0 = im.seg[k].mcu_row_start; sg.my1 = im.seg[k].mcu_row_end;
            for (int c = 0; c < 3; ++c) sg.lastdc[c] = im.seg[k].last_dc[c];
            sg.ov_bits = im.seg[k].overhang_bits; sg.ov_byte = im.seg[k].overhang_byte;
            sg.out_off = off; sg.expect = im.seg[k].expect_bytes; sg.is_last = k + 1 == im.nseg;
            off += im.seg[k].expect_bytes;
            p.segs.push_back(sg);
        }
        p.total += align_up((size_t)im.scan_bytes + 16, 256);
    }
}

}  // namespace lepb200
