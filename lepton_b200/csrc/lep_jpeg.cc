// lep_jpeg.cc -- JPEG front end: marker-level parse, de-stuffing, baseline Huffman decode to coefficient
// planes in the reference's AlignedBlock order, per-MCU-row ThreadHandoff capture.
//
// Behavioural model: read_jpeg (jpgcoder.cc:2270-2466), setup_imginfo_jpg (:4450-4540), parse_jfif_jpg
// (:4545-4800), decode_jpeg (:2799-3302), decode_block_seq (:4893-4961), next_mcupos (recoder.cc:190-243),
// crystallize_thread_handoff (jpgcoder.cc:2520-2560).  The implementation is new (table-driven Huffman decoder
// over a 64-bit window on the de-stuffed stream); files the reference would refuse are refused with the same
// ExitCode, and reference features not covered yet return NOT_HANDLED rather than guessing.
#include <algorithm>
#include <cmath>

#include <cstdio>
#include <cstring>
#include <ctime>

#include "lep_scan.h"

namespace lephost {

namespace {

bool fail(Jpeg& j, int status, const char* msg) {
    j.status = status;
    j.error = msg;
    return false;
}

}  // namespace

bool HuffTable::build() {
    // canonical code assignment (ITU T.81 Annex C); also the encode-side code/length arrays
    int code = 0, k = 0;
    memset(fast, 0, sizeof(fast));
    memset(elen, 0, sizeof(elen));
    memset(ecode, 0, sizeof(ecode));
    for (int len = 1; len <= 16; ++len) {
        valoff[len] = k - code;
        for (int i = 0; i < bits[len]; ++i, ++k, ++code) {
            if (k >= 256 || code >= (1 << len)) return false;        // more codes of this length than the code space holds
            const uint8_t sym = vals[k];
            ecode[sym] = (uint16_t)code;
            elen[sym] = (uint8_t)len;
            if (len <= 9) {
                const int shift = 9 - len;
                for (int f = 0; f < (1 << shift); ++f) fast[(code << shift) | f] = (uint16_t)((len << 8) | sym);
            }
        }
        maxcode[len] = bits[len] ? code - 1 : -1;
        if (code > (1 << len)) return false;
        code <<= 1;
    }
    maxcode[17] = 0x7fffffff;
    // largest end-of-band run this table can express (build_huffcodes, jpgcoder.cc:5542-5549)
    max_eobrun = 0;
    for (int i = 14; i >= 0; --i)
        if (elen[i << 4] > 0) { max_eobrun = (2 << i) - 1; break; }
    return true;
}

// ------------------------------------------------------------------------------------------------
// read_jpeg: split the file into header segments / de-stuffed entropy data / trailing garbage
// ------------------------------------------------------------------------------------------------
bool parse_frame(Jpeg& j);

bool parse_jpeg(const uint8_t* data, size_t n, Jpeg& j, long long embedding, bool discard_meta) {
    size_t pos = 2;                       // jpg_ident_offset (jpgcoder.cc:1809)
    if (embedding < 0) {
        if (n < 4 || data[0] != 0xFF || data[1] != 0xD8) return fail(j, UNSUPPORTED_JPEG, "not a JPEG (no SOI)");
    } else {
        // the reference reads the two bytes that tell the file type, then N more, and keeps the first N of them as the
        // prefix: the JPEG's own SOI is taken on trust (jpgcoder.cc:2275-2281)
        if (n < 2 || (unsigned long long)n - 2 < (unsigned long long)embedding) return fail(j, ASSERTION_FAILURE, "embedding offset beyond the end of the file");
        j.prefix.assign(data, data + embedding);
        pos = (size_t)embedding + 2;
    }
    uint8_t type = 0, seg0 = 0, seg1 = 0;
    bool eof_called = false;
    int scnc = 0;
    j.huff.reserve(n);
    j.hdr.reserve(4096);
    while (true) {
        if (type == 0xDA) {
            unsigned cpos = 0, crst = 0;
            bool scan_done = false;
            while (!scan_done) {
                j.offs.emplace_back((uint32_t)j.huff.size(), (uint32_t)pos);
                if (pos >= n) { j.early_eof = true; eof_called = true; scan_done = true; seg0 = 0; break; }
                uint8_t tmp = data[pos++];
                if (tmp != 0xFF) {
                    crst = 0;
                    // bulk copy of the run of non-FF bytes
                    const uint8_t* run = data + pos - 1;
                    const uint8_t* ff = (const uint8_t*)memchr(run, 0xFF, n - (pos - 1));
                    size_t len = ff ? (size_t)(ff - run) : n - (pos - 1);
                    j.huff.append(run, len);
                    pos = (pos - 1) + len;
                    if (!ff) { j.early_eof = true; eof_called = true; tmp = run[len - 1]; }
                    else { tmp = 0xFF; pos++; }
                }
                if (tmp == 0xFF) {
                    if (pos >= n) { j.early_eof = true; eof_called = true; scan_done = true; seg0 = 0; break; }
                    tmp = data[pos++];
                    if (tmp == 0x00) {
                        crst = 0;
                        j.huff.push_back(0xFF);
                    } else if (tmp == 0xD0 + (cpos & 7)) {
                        cpos++; crst++;
                        while (j.rst_cnt.size() <= (size_t)scnc) j.rst_cnt.push_back(0);
                        ++j.rst_cnt[scnc];
                    } else {
                        if ((int)j.rst_err.size() < scnc) j.rst_err.insert(j.rst_err.end(), scnc - j.rst_err.size(), 0);
                        j.rst_err.push_back((uint8_t)crst);
                        scnc++;
                        seg0 = 0xFF; seg1 = tmp;
                        scan_done = true;
                    }
                } else {
                    scan_done = true;      // end of file inside the scan
                    seg0 = 0;
                }
            }
            if (j.early_eof) break;
        } else {
            if (pos + 2 > n) break;
            seg0 = data[pos]; seg1 = data[pos + 1];
            pos += 2;
            if (seg0 != 0xFF) return fail(j, UNSUPPORTED_JPEG, "size mismatch in marker segment");
        }
        type = seg1;
        if (type == 0xD9) { eof_called = true; break; }
        if (pos + 2 > n) break;
        const unsigned len = 2 + be16(data + pos);
        if (len < 4) break;
        if (pos + (len - 2) > n) break;
        // segment = FF type len_hi len_lo payload
        j.hdr.push_back(0xFF); j.hdr.push_back(type);
        j.hdr.insert(j.hdr.end(), data + pos, data + pos + (len - 2));
        pos += len - 2;
    }
    if (!eof_called || j.hdr.empty()) return fail(j, UNSUPPORTED_JPEG, "unexpected end of data encountered in header");
    if (j.huff.empty()) return fail(j, UNSUPPORTED_JPEG, "unexpected end of data encountered in huffman");
    if (j.huff.overflow) return fail(j, ASSERTION_FAILURE, "entropy staging buffer too small");
    // garbage: the last two bytes read, then the rest of the file (jpgcoder.cc:2429-2447)
    {
        uint8_t g0 = pos >= 2 ? data[pos - 2] : 0, g1 = pos >= 1 ? data[pos - 1] : 0;
        j.grb.push_back(g0); j.grb.push_back(g1);
        j.grb.insert(j.grb.end(), data + pos, data + n);
        if (j.grb.size() == 2 && j.grb[0] == 0xFF && j.grb[1] == 0xD9) j.grb.clear();
    }
    j.filesize = (uint32_t)n;
    if (!parse_frame(j)) return false;
    // -d: the reference drops the other segments when it writes the container (write_ujpg, jpgcoder.cc:3797-3800); the
    // decode never reads them, so they can go here
    if (discard_meta) j.hdr = coding_segments(j.hdr);
    return true;
}

// setup_imginfo_jpg + the SOF/DQT cases of parse_jfif_jpg
bool parse_frame(Jpeg& j) {
    size_t hpos = 0;
    const std::vector<uint8_t>& h = j.hdr;
    while (hpos + 4 <= h.size()) {
        const uint8_t type = h[hpos + 1];
        const size_t len = 2 + be16(&h[hpos + 2]);
        if (hpos + len > h.size()) return fail(j, UNSUPPORTED_JPEG, "truncated header segment");      // the header of a .lep is untrusted input
        const uint8_t* seg = &h[hpos];
        if (type == 0xDB) {
            size_t p = 4;
            while (p < len) {
                const int pq = seg[p] >> 4, tq = seg[p] & 15;
                if (pq >= 2 || tq >= 4) break;
                ++p;
                if (pq == 0) {
                    for (int i = 0; i < 64; ++i) {
                        j.qtables[tq][i] = p + i < len ? seg[p + i] : 0;
                        if (j.qtables[tq][i] == 0) break;          // reference quirk: stops at the first zero (jpgcoder.cc:4602)
                    }
                    p += 64;
                } else {
                    for (int i = 0; i < 64; ++i) {
                        j.qtables[tq][i] = p + 2 * i + 1 < len ? (uint16_t)be16(seg + p + 2 * i) : 0;
                        if (j.qtables[tq][i] == 0) break;
                    }
                    p += 128;
                }
                j.qt_set[tq] = true;
            }
            if (p != len) return fail(j, UNSUPPORTED_JPEG, "size mismatch in dqt marker");
        } else if (type == 0xC0 || type == 0xC1 || type == 0xC2) {
            j.jpegtype = type == 0xC2 ? 2 : 1;
            if (len < 10) return fail(j, UNSUPPORTED_JPEG, "short SOF");
            if (seg[4] != 8) return fail(j, UNSUPPORTED_JPEG, "data precision not supported");
            j.height = be16(seg + 5);
            j.width = be16(seg + 7);
            j.ncmp = seg[9];
            if (j.ncmp > 4) return fail(j, UNSUPPORTED_JPEG, "too many components");
            if (len < (size_t)(10 + 3 * j.ncmp)) return fail(j, UNSUPPORTED_JPEG, "short SOF");
            for (int c = 0; c < j.ncmp; ++c) {
                Component& k = j.cmp[c];
                k.jid = seg[10 + 3 * c];
                k.H = seg[11 + 3 * c] >> 4;
                k.V = seg[11 + 3 * c] & 15;
                if (k.H > 4 || k.V > 4) return fail(j, 11 /*SAMPLING_BEYOND_FOUR_UNSUPPORTED*/, "sampling factor > 4");
                if (k.H > 2 || k.V > 2) return fail(j, SAMPLING_BEYOND_TWO_UNSUPPORTED, "sampling factor > 2");
                k.tq = seg[12 + 3 * c];
                if (k.tq >= 4) return fail(j, UNSUPPORTED_JPEG, "bad quantisation table id");
            }
        } else if (type == 0xC3 || (type >= 0xC5 && type <= 0xC7) || (type >= 0xC9 && type <= 0xCB) || (type >= 0xCD && type <= 0xCF)) {
            return fail(j, UNSUPPORTED_JPEG, "unsupported SOF type (lossless / differential / arithmetic)");
        }
        hpos += len;
    }
    if (j.ncmp == 0 || j.jpegtype == 0) return fail(j, UNSUPPORTED_JPEG, "header contains incomplete information");
    if (j.ncmp > 3) return fail(j, UNSUPPORTED_4_COLORS, "4 colour channels");
    int hm = 0, vm = 0;
    for (int c = 0; c < j.ncmp; ++c) {
        const Component& k = j.cmp[c];
        if (k.H == 0 || k.V == 0 || !j.qt_set[k.tq] || j.qtables[k.tq][0] == 0) return fail(j, UNSUPPORTED_JPEG, "header information is incomplete");
        hm = std::max(hm, k.H); vm = std::max(vm, k.V);
    }
    j.mcuv = (int)std::ceil((float)j.height / (float)(8 * vm));
    j.mcuh = (int)std::ceil((float)j.width / (float)(8 * hm));
    j.mcuc = j.mcuv * j.mcuh;
    if (j.mcuc <= 0) return fail(j, UNSUPPORTED_JPEG, "empty image");
    for (int c = 0; c < j.ncmp; ++c) {
        Component& k = j.cmp[c];
        k.mbs = k.H * k.V;
        k.bcv = j.mcuv * k.V;
        k.bch = j.mcuh * k.H;
        k.bc = k.bcv * k.bch;
        k.ncv = (int)std::ceil((float)j.height * ((float)k.V / (8.0 * vm)));
        k.nch = (int)std::ceil((float)j.width * ((float)k.H / (8.0 * hm)));
    }
    return true;
}

// Quick marker walk up to the first SOF: total bytes of the coefficient planes (0 if not determinable here;
// the full parse then reports the precise error).  Used to lay out the pinned plane arena before decoding.
size_t peek_plane_bytes(const uint8_t* data, size_t n, long long embedding) {
    size_t pos = 2;
    if (embedding < 0) {
        if (n < 4 || data[0] != 0xFF || data[1] != 0xD8) return 0;
    } else {
        if ((unsigned long long)n < (unsigned long long)embedding + 2) return 0;
        pos = (size_t)embedding + 2;
    }
    while (pos + 4 <= n) {
        if (data[pos] != 0xFF) return 0;
        const uint8_t type = data[pos + 1];
        if (type == 0xD9 || type == 0xDA) return 0;
        const size_t len = 2 + be16(data + pos + 2);
        if (type == 0xC0 || type == 0xC1 || type == 0xC2) {
            if (pos + len > n || len < 10) return 0;
            const uint8_t* seg = data + pos;
            const int height = be16(seg + 5), width = be16(seg + 7), nc = seg[9];
            if (nc < 1 || nc > 4 || len < (size_t)(10 + 3 * nc)) return 0;
            int hm = 0, vm = 0;
            for (int c = 0; c < nc; ++c) { hm = std::max(hm, seg[11 + 3 * c] >> 4); vm = std::max(vm, seg[11 + 3 * c] & 15); }
            if (!hm || !vm) return 0;
            const size_t mcuv = (size_t)std::ceil((float)height / (float)(8 * vm)), mcuh = (size_t)std::ceil((float)width / (float)(8 * hm));
            size_t total = 0;
            for (int c = 0; c < nc; ++c) {
                const size_t pb = mcuv * (seg[11 + 3 * c] & 15) * mcuh * (seg[11 + 3 * c] >> 4) * 128;
                total += (pb + 255) & ~size_t(255);
            }
            return total;
        }
        pos += len;
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Huffman decoding
// ------------------------------------------------------------------------------------------------
namespace {

struct BitReader {
    const uint8_t* d;
    size_t n;          // bytes
    uint64_t bitpos;   // bits consumed
    bool at_eof = false;   // abitreader::eof (bitops.hh:262-306): set by the read that consumes the last bit (or tries to go past it)
    inline bool eof() const { return at_eof; }
    // peek 32 bits at the current position (zero beyond the end)
    inline uint32_t peek32() const {
        size_t byte = (size_t)(bitpos >> 3);
        uint64_t v = 0;
        if (byte + 8 <= n) {
            uint64_t raw;
            memcpy(&raw, d + byte, 8);
            v = __builtin_bswap64(raw);
        } else {
            for (int i = 0; i < 8; ++i) v = (v << 8) | (byte + i < n ? d[byte + i] : 0);
        }
        return (uint32_t)((v << (bitpos & 7)) >> 32);
    }
    inline void skip(int k) {
        if (!k) return;
        if (bitpos + (uint64_t)k >= (uint64_t)n * 8) { at_eof = true; bitpos = (uint64_t)n * 8; }
        else bitpos += (uint64_t)k;
    }
    // >= 57 valid bits at the current position, MSB first (zero beyond the end)
    inline uint64_t peek57() const {
        size_t byte = (size_t)(bitpos >> 3);
        uint64_t v = 0;
        if (byte + 8 <= n) {
            uint64_t raw;
            memcpy(&raw, d + byte, 8);
            v = __builtin_bswap64(raw);
        } else {
            for (int i = 0; i < 8; ++i) v = (v << 8) | (byte + i < n ? d[byte + i] : 0);
        }
        return v << (bitpos & 7);
    }
};

// One Huffman symbol plus its magnitude bits from a single 57-bit window (code <= 16 bits, magnitude <= 16 bits).
// Returns the symbol (-1 on an invalid code); *value receives DEVLI(size, bits) where size = symbol & mask.
inline int decode_symbol_value(BitReader& br, const HuffTable& t, int size_mask, int* value) {
    const uint64_t win = br.peek57();
    const uint16_t f = t.fast[win >> 55];
    int len, sym;
    if (f) { len = f >> 8; sym = f & 0xff; }
    else {
        const uint32_t w = (uint32_t)(win >> 32);
        int code = (int)(w >> 22);
        len = 10;
        while (len <= 16 && code > t.maxcode[len]) { ++len; code = (int)(w >> (32 - len)); }
        if (len > 16) return -1;
        sym = t.vals[code + t.valoff[len]];
    }
    const int s = sym & size_mask;
    int v = 0;
    const uint64_t p = br.bitpos + (uint64_t)len, end = (uint64_t)br.n * 8, tail = (uint64_t)(br.n & ~(size_t)7) * 8;
    if (s && (br.n & 7) && p < tail && p + (uint64_t)s > end) {
        // Magnitude bits that run past the end of truncated data across the start of its last, partial 8-byte word.
        // The reference's abitreader loads the data 8 bytes at a time; a read that needs more bits than that last
        // load holds takes them right-aligned (bitops.hh:294-301), so the missing bits sit between the two parts, not
        // at the end, and eof is only set by the next read (the reader is left at the end, not yet at eof).
        const int k = (int)(tail - p);
        uint32_t lastw = 0;
        for (size_t i = br.n & ~(size_t)7; i < br.n; ++i) lastw = (lastw << 8) | br.d[i];
        const int nb = (int)((((win << len) >> (64 - k)) << (s - k)) | lastw) & (int)((1u << s) - 1u);
        *value = nb >= (1 << (s - 1)) ? nb : (int)((unsigned)nb + 1u - (1u << s));
        br.bitpos = end;
        return sym;
    }
    if (s) {
        const int nb = (int)((win << len) >> (64 - s));
        v = nb >= (1 << (s - 1)) ? nb : (int)((unsigned)nb + 1u - (1u << s));     // unsigned: a DC size up to 31 (refused by the caller) must not overflow
    }
    *value = v;
    br.skip(len + s);
    return sym;
}

// one Huffman symbol; -1 on invalid code / read past the end
inline int decode_symbol(BitReader& br, const HuffTable& t) {
    const uint32_t w = br.peek32();
    const uint16_t f = t.fast[w >> 23];
    if (f) {
        br.skip(f >> 8);
        return f & 0xff;
    }
    int code = (int)(w >> 22);   // 10 bits
    int len = 10;
    while (len <= 16 && code > t.maxcode[len]) { ++len; code = (int)(w >> (32 - len)); }
    if (len > 16) return -1;
    br.skip(len);
    return t.vals[code + t.valoff[len]];
}

inline int devli(int s, int n) { return s == 0 ? n : (n >= (1 << (s - 1)) ? n : n + 1 - (1 << s)); }

// crystallize_thread_handoff (jpgcoder.cc:2520-2560).  abitreader::getpos() == (bits consumed >> 3) + 1.
Handoff crystallize(const Jpeg& j, const BitReader& br, int mcu_y, const int lastdc[4], int luma_mul) {
    const uint32_t gp = (uint32_t)(br.bitpos >> 3) + 1;
    const auto& offs = j.offs;
    auto it = std::lower_bound(offs.begin(), offs.end(), std::pair<uint32_t, uint32_t>(gp, gp));
    if (it != offs.begin()) --it;
    uint32_t mapped = 0;
    if (it != offs.end()) mapped = it->second + (gp - it->first);
    Handoff h;
    h.segment_size = mapped;
    for (int i = 0; i < 3; ++i) h.last_dc[i] = (int16_t)lastdc[i];
    h.luma_y_start = (uint16_t)(luma_mul * mcu_y);
    h.luma_y_end = (uint16_t)(luma_mul * (mcu_y + 1));
    const int rem = (int)(br.bitpos & 7);
    h.num_overhang_bits = (uint8_t)rem;
    uint8_t cur = (size_t)(br.bitpos >> 3) < br.n ? br.d[br.bitpos >> 3] : 0;
    h.overhang_byte = (uint8_t)(cur & (((1 << rem) - 1) << (8 - rem)));
    return h;
}

// abitreader::unpad (bitops.hh:316-332)
int8_t unpad(BitReader& br, int8_t fillbit) {
    if ((br.bitpos & 7) == 0 || br.eof()) return fillbit;
    auto rd = [&]() { int b = br.eof() ? 0 : (br.d[br.bitpos >> 3] >> (7 - (br.bitpos & 7))) & 1; br.skip(1); return b; };
    int last = rd();
    int fb = last, offset = 1;
    while (br.bitpos & 7) { last = rd(); fb |= last << offset; ++offset; }
    while (offset < 7) { fb |= last << offset; ++offset; }
    return (int8_t)fb;
}

// read k (<= 16) raw bits, MSB first; zero past the end (abitreader::read, bitops.hh:262-306)
inline int read_bits(BitReader& br, int k) {
    if (!k) return 0;
    const int v = (int)(br.peek32() >> (32 - k));
    br.skip(k);
    return v;
}

// skip_eobrun (jpgcoder.cc:5462-5503): jump over the blocks an end-of-band run covers
inline int skip_eobrun(const Jpeg& j, int rsti, ScanPos& p, unsigned& eobrun) {
    if (eobrun == 0) return 0;
    const Component& k = j.cmp[p.cmp];
    if (rsti > 0) {
        if ((int)eobrun > p.rstw) return -1;
        p.rstw -= (int)eobrun;
    }
    if (k.bch != k.nch) p.dpos += (int)(((unsigned)(p.dpos % k.bch) + eobrun) / (unsigned)k.nch) * (k.bch - k.nch);
    if (k.bcv != k.ncv && p.dpos / k.bch >= k.ncv) p.dpos += (k.bcv - k.ncv) * k.bch;
    p.dpos += (int)eobrun;
    eobrun = 0;
    if (p.dpos == k.bc) return 2;
    if (p.dpos > k.bc) return -1;
    if (rsti > 0 && p.rstw == 0) return 1;
    return 0;
}

// One restart interval of a progressive scan (decode_jpeg, jpgcoder.cc:2985-3258; block routines :4968-5340).
// Returns the reference's `sta` (1 restart, 2 scan done, -1 error); handoffs are recorded only by first-stage DC scans.
int decode_progressive_interval(Jpeg& j, BitReader& br, const ScanInfo& sc, const ScanTables& t,
                                int16_t* const planes[4], ScanPos& p, int lastdc[4], bool& handoff_due, int luma_mul) {
    const int rsti = t.rsti;
    int sta = 0;
    unsigned eobrun = 0, peobrun = 0;
    auto track = [&]() { if (!br.eof()) j.max_dpos[p.cmp] = std::max(j.max_dpos[p.cmp], p.dpos); };
    auto coef = [&](int bpos) -> int16_t& { return planes[p.cmp][(size_t)p.dpos * 64 + k_zigzag_to_aligned[bpos]]; };
    if (sc.ncomp > 1 || sc.to == 0) {
        const bool inter = sc.ncomp > 1;
        if (sc.sah == 0) {
            // ---- DC, first stage (decode_dc_prg_fs :4968)
            while (sta == 0) {
                if (handoff_due) {
                    j.rows.push_back(crystallize(j, br, inter ? p.mcu / j.mcuh : p.dpos / j.cmp[p.cmp].bch, lastdc, luma_mul));
                    handoff_due = false;
                }
                track();
                int diff = 0;
                const int s = decode_symbol_value(br, t.dc[t.td[p.cmp]], 0x1f, &diff);
                if (s < 0 || s > 16) { sta = -1; diff = 0; }
                const int16_t v = (int16_t)(diff + lastdc[p.cmp]);
                lastdc[p.cmp] = v;
                coef(0) = (int16_t)((uint16_t)v << sc.sal);
                if (inter) {
                    const int old_mcu = p.mcu;
                    if (sta != -1) sta = next_mcupos(j, sc, rsti, p);
                    if (p.mcu % j.mcuh == 0 && old_mcu != p.mcu) handoff_due = true;
                } else {
                    if (sta != -1) sta = next_mcuposn(j, rsti, p);
                    if (p.cmp == 0 && p.dpos % j.cmp[p.cmp].bch == 0) handoff_due = true;
                }
                if (br.eof()) { sta = 2; break; }
            }
        } else {
            // ---- DC refinement: one bit per block (decode_dc_prg_sa :5124)
            while (sta == 0) {
                track();
                const int bit = read_bits(br, 1);
                coef(0) = (int16_t)(coef(0) + (bit << sc.sal));
                sta = inter ? next_mcupos(j, sc, rsti, p) : next_mcuposn(j, rsti, p);
                if (br.eof()) { sta = 2; break; }
            }
        }
        return sta;
    }
    const HuffTable& act = t.ac[t.ta[p.cmp]];
    if (sc.sah == 0) {
        // ---- AC, first stage (decode_ac_prg_fs :5014)
        while (sta == 0) {
            track();
            int eob = sc.to + 1;
            if (eobrun > 0) {
                --eobrun;                                  // the block stays as it is (copy loop :3178 is empty)
                eob = sc.from;
            } else {
                int bpos = sc.from;
                while (bpos <= sc.to) {
                    int v = 0;
                    const int hc = decode_symbol_value(br, act, 0, &v);     // magnitude bits read below (depends on the symbol class)
                    if (hc < 0) { eob = -1; break; }
                    const int l = hc >> 4, r = hc & 15;
                    if (l == 15 || r > 0) {
                        const int n = read_bits(br, r);
                        if (l + bpos > sc.to) { eob = -1; break; }
                        for (int z = 0; z < l; ++z) coef(bpos++) = 0;
                        coef(bpos++) = (int16_t)((uint16_t)(int16_t)devli(r, n) << sc.sal);
                    } else {
                        eob = bpos;
                        const int n = read_bits(br, l);
                        eobrun = (unsigned)(n + (1 << l));
                        --eobrun;
                        break;
                    }
                }
            }
            if (eob == sc.from && eobrun > 0 && peobrun > 0 && peobrun < (unsigned)act.max_eobrun - 1) {
                j.status = ASSERTION_FAILURE; j.error = "reconstruction of non optimal coding not supported";   // errorlevel 1
            }
            if (eob < 0) sta = -1;
            else sta = skip_eobrun(j, rsti, p, eobrun);
            if (sta == 0) sta = next_mcuposn(j, rsti, p);
            if (br.eof()) { sta = 2; break; }
        }
        return sta;
    }
    // ---- AC refinement (decode_ac_prg_sa :5150, decode_eobrun_sa :5322), in place: the reference copies the band into a
    // scratch block, replaces every already non-zero coefficient by its correction bit and adds the scratch block back
    // shifted; here the same additions are applied directly, and the already non-zero coefficients of the block come
    // from one vector compare (zig-zag-ordered bit mask) instead of 63 loads -- these scans visit every block of a
    // component and dominate the decode time of progressive files.
    const uint64_t band = (sc.to >= 63 ? ~0ull : ((1ull << (sc.to + 1)) - 1)) & ~((1ull << sc.from) - 1);
    auto correct = [&](int z) {                    // one correction bit for the non-zero coefficient at zig-zag position z
        if (read_bits(br, 1)) {
            int16_t& cf = coef(z);
            cf = (int16_t)(cf + (int16_t)((uint16_t)(int16_t)(cf > 0 ? 1 : -1) << sc.sal));
        }
    };
    auto correct_all = [&](uint64_t m) {           // correction bits of all coefficients in m, ascending zig-zag order, read in batches
        while (m) {
            const int k = std::min(__builtin_popcountll(m), 24);
            const uint32_t bits = (uint32_t)read_bits(br, k);          // first coefficient's bit on top
            for (int i = k - 1; i >= 0; --i) {
                const int z = __builtin_ctzll(m);
                m &= m - 1;
                if ((bits >> i) & 1u) {
                    int16_t& cf = coef(z);
                    cf = (int16_t)(cf + (int16_t)((uint16_t)(int16_t)(cf > 0 ? 1 : -1) << sc.sal));
                }
            }
        }
    };
    while (sta == 0) {
        const uint64_t nzm = nonzero_mask_zigzag(planes[p.cmp] + (size_t)p.dpos * 64) & band;
        int eob = sc.to;
        track();
        if (eobrun == 0) {
            int bpos = sc.from;
            bool err = false;
            while (bpos <= sc.to) {
                int dummy = 0;
                const int hc = decode_symbol_value(br, act, 0, &dummy);
                if (hc < 0) { err = true; break; }
                const int l = hc >> 4, r = hc & 15;
                if (l == 15 || r > 0) {
                    int z = l, v = 0;
                    if (r == 1) v = read_bits(br, 1) ? 1 : -1;
                    else if (r != 0) { err = true; break; }
                    while (true) {
                        if (!((nzm >> bpos) & 1)) {
                            if (z > 0) --z;
                            else {
                                if (v) coef(bpos) = (int16_t)((uint16_t)(int16_t)v << sc.sal);
                                ++bpos;
                                break;
                            }
                        } else {
                            correct(bpos);
                        }
                        if (bpos++ >= sc.to) { err = true; break; }
                    }
                    if (err) break;
                } else {
                    eob = bpos;
                    const int n = read_bits(br, l);
                    eobrun = (unsigned)(n + (1 << l));
                    break;
                }
            }
            if (err) eob = -1;
            else if (eobrun > 0) {
                correct_all(bpos <= 63 ? nzm & ~((1ull << bpos) - 1) : 0ull);
                --eobrun;
            }
            if (eob == sc.from && eobrun > 0 && peobrun > 0 && peobrun < (unsigned)act.max_eobrun - 1) {
                j.status = ASSERTION_FAILURE; j.error = "reconstruction of non optimal coding not supported";
            }
        } else {
            correct_all(nzm);
            --eobrun;
            eob = 0;
        }
        peobrun = eobrun;
        if (eob < 0) sta = -1;
        else sta = next_mcuposn(j, rsti, p);
        if (br.eof()) { sta = 2; break; }
    }
    return sta;
}

}  // namespace

// ThreadHandoff for a Huffman state captured elsewhere (the GPU decoder): same mapping as crystallize().
Handoff handoff_from_state(const Jpeg& j, uint32_t bitpos, int mcu_y, const int16_t lastdc[3]) {
    BitReader br{j.huff.data(), j.huff.size(), bitpos, false};
    int ldc[4] = {lastdc[0], lastdc[1], lastdc[2], 0};
    return crystallize(j, br, mcu_y, ldc, j.cmp[0].bcv / j.mcuv);
}

// Single-scan baseline set-up for the GPU Huffman decoder: tables chosen by the SOS, restart interval.  Returns false
// (without touching j.status) when the file needs the general host path (progressive, truncated, several scans, scan
// order != frame order, a header the host refuses).
bool gpu_scan_setup(const Jpeg& j, GpuScanSetup& out, size_t* sos_end) {
    if (j.jpegtype != 1 || j.early_eof || j.ncmp < 1 || j.ncmp > 3) return false;   // truncated files take the host path
    ScanTables t;
    ScanInfo sc;
    const char* err = nullptr;
    size_t pos = 0;
    if (read_to_sos(j, pos, t, sc, err) != Seg::sos || sc.ncomp != j.ncmp || !scan_tables_present(j, t, sc)) return false;
    for (int i = 0; i < sc.ncomp; ++i) if (sc.cmp[i] != i) return false;          // scan order must be frame order
    const size_t end = pos;
    const int ndef = t.ndef;
    ScanInfo next;
    if (read_to_sos(j, pos, t, next, err) != Seg::end || t.ndef != ndef) return false;   // one scan, no tables behind it
    out.rsti = t.rsti;
    for (int c = 0; c < j.ncmp; ++c) {
        memcpy(out.dc[c].bits, t.dc[t.td[c]].bits, 17); memcpy(out.dc[c].vals, t.dc[t.td[c]].vals, 256);
        memcpy(out.ac[c].bits, t.ac[t.ta[c]].bits, 17); memcpy(out.ac[c].vals, t.ac[t.ta[c]].vals, 256);
    }
    if (sos_end) *sos_end = end;
    return true;
}

bool decode_scans(Jpeg& j, int16_t* const planes[4]) {
    ScanTables t;
    BitReader br{j.huff.data(), j.huff.size(), 0, false};
    int lastdc[4] = {0, 0, 0, 0};
    size_t hpos = 0;
    const int luma_mul = j.cmp[0].bcv / j.mcuv;
    int mcu = 0;
    int scans = 0;
    j.padbit = -1;
    j.is_baseline = true;
    while (true) {
        ScanInfo sc;
        const char* err = nullptr;
        const Seg seg = read_to_sos(j, hpos, t, sc, err);
        if (seg == Seg::error) return fail(j, UNSUPPORTED_JPEG, err);
        if (seg == Seg::end) break;
        if (!scan_tables_present(j, t, sc)) return fail(j, UNSUPPORTED_JPEG, "huffman table missing in scan");
        const int rsti = t.rsti;
        if (sc.ncomp != j.ncmp || j.jpegtype != 1) j.is_baseline = false;     // jpgcoder.cc:2912-2926: written with flag 'X'
        ScanPos p;
        p.cmp = sc.cmp[0];
        if (!br.eof()) {                              // jpgcoder.cc:2879-2886
            j.max_bpos = std::max(j.max_bpos, sc.to);
            j.max_sah = std::max(j.max_sah, std::max(sc.sal, sc.sah));
            for (int i = 0; i < sc.ncomp; ++i) j.max_cmp = std::max(j.max_cmp, sc.cmp[i]);
        }
        bool handoff_due = true;
        if (j.jpegtype != 1) {
#ifdef LEPB200_SCAN_TIMING
            timespec ts0; clock_gettime(CLOCK_MONOTONIC, &ts0);
#endif
            mcu = 0;
            while (true) {
                lastdc[0] = lastdc[1] = lastdc[2] = lastdc[3] = 0;
                p.rstw = rsti;
                const int sta = decode_progressive_interval(j, br, sc, t, planes, p, lastdc, handoff_due, luma_mul);
                if (j.status != OK) return false;
                if (j.padbit != -1) {
                    if (j.padbit != unpad(br, j.padbit)) return fail(j, UNSUPPORTED_JPEG, "inconsistent use of padbits");
                } else {
                    j.padbit = unpad(br, j.padbit);
                }
                if (sta == -1) return fail(j, UNSUPPORTED_JPEG, "decode error in progressive scan");
                if (sta == 2) { ++scans; break; }
            }
            if (sc.ncomp > 1) mcu = p.mcu;              // the last handoff is taken at mcu / mcuh (jpgcoder.cc:3278)
#ifdef LEPB200_SCAN_TIMING
            { timespec ts1; clock_gettime(CLOCK_MONOTONIC, &ts1);
              fprintf(stderr, "[scan] ncomp %d cmp %d Ss %d Se %d Ah %d Al %d  %.1f ms\n", sc.ncomp, sc.cmp[0], sc.from, sc.to, sc.sah, sc.sal,
                      (ts1.tv_sec - ts0.tv_sec) * 1e3 + (ts1.tv_nsec - ts0.tv_nsec) * 1e-6); }
#endif
            continue;
        }

        int sta = 0;
        const int hmul = j.cmp[0].bch / j.mcuh, vmul = j.cmp[0].bcv / j.mcuv;
        while (true) {
            lastdc[0] = lastdc[1] = lastdc[2] = lastdc[3] = 0;
            sta = 0;
            p.rstw = rsti;
            while (sta == 0) {
                if (handoff_due) {
                    j.rows.push_back(crystallize(j, br, p.mcu / j.mcuh, lastdc, luma_mul));
                    handoff_due = false;
                }
                if (!br.eof()) j.max_dpos[p.cmp] = std::max(j.max_dpos[p.cmp], p.dpos);     // jpgcoder.cc:2941-2943
                // ---- decode_block_seq
                const HuffTable& dct = t.dc[t.td[p.cmp]];
                const HuffTable& act = t.ac[t.ta[p.cmp]];
                int16_t* blk = planes[p.cmp] + (size_t)p.dpos * 64;
                int dcdiff = 0;
                int s = decode_symbol_value(br, dct, 0x1f, &dcdiff);
                if (s < 0 || s > 16) return fail(j, UNSUPPORTED_JPEG, "decode error in scan (dc)");
                int16_t dcv = (int16_t)(dcdiff + lastdc[p.cmp]);
                lastdc[p.cmp] = dcv;
                blk[k_zigzag_to_aligned[0]] = dcv;
                int bpos = 1, eob = 64;
                int last_nonzero_written = 1;   // whether block[eob-1] != 0 (reference check :2953)
                while (bpos < 64) {
                    int v = 0;
                    int hc = decode_symbol_value(br, act, 15, &v);
                    if (hc < 0) return fail(j, UNSUPPORTED_JPEG, "decode error in scan (ac)");
                    if (hc > 0) {
                        int z = hc >> 4;
                        if (z + bpos >= 64) {
                            // eof_fixup (jpgcoder.cc:4930-4958): only legal when the data ran out; the rest of the block
                            // is zero and the last coefficient is set to 1 so that the block has no trailing zero run
                            if (!br.eof()) return fail(j, ASSERTION_FAILURE, "zero run longer than the block in complete data");
                            for (int q = bpos; q < 64; ++q) blk[k_zigzag_to_aligned[q]] = 0;
                            blk[k_zigzag_to_aligned[63]] = 1;
                            last_nonzero_written = 1;
                            eob = 64;
                            break;
                        }
                        bpos += z;
                        blk[k_zigzag_to_aligned[bpos++]] = (int16_t)v;
                        last_nonzero_written = v != 0;
                    } else {
                        eob = bpos;
                        break;
                    }
                }
                if (eob > 1 && !last_nonzero_written) return fail(j, UNSUPPORTED_JPEG, "cannot encode image with eob after last 0");
                // ---- next position
                if (sc.ncomp > 1) {
                    const int old_mcu = p.mcu;
                    sta = next_mcupos(j, sc, rsti, p);
                    if (p.mcu % j.mcuh == 0 && old_mcu != p.mcu) handoff_due = true;
                } else {
                    sta = next_mcuposn(j, rsti, p);
                    p.mcu = p.dpos / (hmul * vmul);
                    if (p.cmp == 0 && (p.mcu % j.mcuh == 0) && (p.dpos % (hmul * vmul) == 0)) handoff_due = true;
                }
                if (br.eof()) { sta = 2; break; }
            }
            // padbit bookkeeping (jpgcoder.cc:3260-3271)
            if (j.padbit != -1) {
                if (j.padbit != unpad(br, j.padbit)) return fail(j, UNSUPPORTED_JPEG, "inconsistent use of padbits");
            } else {
                j.padbit = unpad(br, j.padbit);
            }
            if (sta == 2) { ++scans; break; }
        }
        mcu = p.mcu;
    }
    if (scans == 0) return fail(j, UNSUPPORTED_JPEG, "no scan found");
    for (int c = 0; c < j.ncmp; ++c) { j.trunc_bcv[c] = j.cmp[c].bcv; j.trunc_bc[c] = j.cmp[c].bc; }
    if (j.early_eof) {
        // UncompressedComponents::set_truncation_bounds / set_block_count_dpos (uncompressed_components.hh:166-188)
        for (int c = 0; c < j.ncmp; ++c) {
            const Component& k = j.cmp[c];
            const int tbc = j.max_dpos[c] + 1;
            int vs = std::min(tbc / k.bch + (tbc % k.bch ? 1 : 0), k.bcv);
            const int ratio = k.bcv / j.mcuv;
            while (vs % ratio != 0 && vs + 1 <= k.bcv) ++vs;
            j.trunc_bcv[c] = vs;
            j.trunc_bc[c] = tbc;
        }
    }
    j.rows.push_back(crystallize(j, br, (uint16_t)(mcu / j.mcuh), lastdc, luma_mul));
    for (size_t i = 1; i < j.rows.size(); ++i)
        if (j.rows[i].luma_y_start < j.rows[i - 1].luma_y_end) j.rows[i].luma_y_start = j.rows[i - 1].luma_y_end;
    if (!br.eof()) return fail(j, UNSUPPORTED_JPEG, "unneeded data found after coded image data");
    return true;
}

}  // namespace lephost
