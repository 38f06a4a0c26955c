// lep_host.h -- host-side (CPU, C++) halves of the drop-in: JPEG front end, .lep container, mux.
//
// These are the callers on either side of the GPU hot path (SURVEY.md section 8(f) "next" rows, host versions):
//   JPEG bytes --parse_jpeg/decode_scans--> coefficient planes + per-MCU-row handoffs
//              --select_splits------------> thread-segments          (reference write_ujpg, jpgcoder.cc:3860-3934)
//              --[GPU: lepb200_encode_*]--> per-segment bool-coder streams
//              --write_lep----------------> .lep bytes               (reference write_ujpg + vp8_full_encoder tail)
// and the inverse for decode.  Everything here must be byte-exact with the reference; citations are to
// /root/reference/src/lepton/jpgcoder.cc unless stated otherwise.
#pragma once
#include "../../include/lepton_b200.h"
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <utility>
#include <vector>

namespace lephost {

// reference ExitCode values used as status (src/vp8/util/memory.hh:13-39) + local "not handled by this build" codes
enum Status : int32_t {
    OK = 0,
    ASSERTION_FAILURE = 1,
    SHORT_READ = 3,
    UNSUPPORTED_4_COLORS = 4,
    COEFFICIENT_OUT_OF_RANGE = 6,
    STREAM_INCONSISTENT = 7,
    PROGRESSIVE_UNSUPPORTED = 8,
    SAMPLING_BEYOND_TWO_UNSUPPORTED = 10,
    THREADING_PARTIAL_MCU = 12,
    VERSION_UNSUPPORTED = 13,
    UNSUPPORTED_JPEG = 42,
    UNSUPPORTED_JPEG_WITH_ZERO_IDCT_0 = 43,
    NOT_HANDLED = 200   // feature of the reference this build does not cover yet (never a silent wrong answer)
};

// ThreadHandoff (src/lepton/thread_handoff.hh:8-39)
struct Handoff {
    uint16_t luma_y_start = 0, luma_y_end = 0;
    uint32_t segment_size = 0;
    uint8_t overhang_byte = 0, num_overhang_bits = 0;
    int16_t last_dc[4] = {0, 0, 0, 0};
    uint32_t tokens = 0;      // not part of the format: decision-count bound of everything before this row (GPU Huffman decoder)
};

struct Component {
    int jid = 0, H = 0, V = 0, tq = 0;                   // H = horizontal sampling (reference "sfv"), V = vertical ("sfh")
    int bch = 0, bcv = 0, bc = 0, nch = 0, ncv = 0, mbs = 0;
};

struct HuffTable {
    bool set = false;
    uint8_t bits[17] = {0};
    uint8_t vals[256] = {0};
    // decode acceleration
    uint16_t fast[512] = {0};  // (len << 8) | symbol for codes of <= 9 bits, 0 = slow path
    int32_t maxcode[18] = {0}; // canonical decode
    int32_t valoff[18] = {0};
    // encode side
    uint16_t ecode[256] = {0};
    uint8_t elen[256] = {0};
    int max_eobrun = 0;        // progressive: longest end-of-band run with a code in this table
    bool build();
};

// De-stuffed entropy-coded bytes of all scans.  Owns its storage by default; attach() makes it write into caller-provided
// memory instead (the file pipeline points it at the pinned staging buffer the GPU Huffman decoder uploads from, so the
// bytes are written exactly once).
struct HuffBuf {
    std::vector<uint8_t> own;
    uint8_t* ext = nullptr;
    size_t ext_cap = 0, ext_n = 0;
    bool overflow = false;
    void attach(uint8_t* p, size_t cap) { ext = p; ext_cap = cap; ext_n = 0; overflow = false; }
    const uint8_t* data() const { return ext ? ext : own.data(); }
    size_t size() const { return ext ? ext_n : own.size(); }
    bool empty() const { return size() == 0; }
    void reserve(size_t n) { if (!ext) own.reserve(n); }
    void clear() { if (ext) ext_n = 0; else own.clear(); }
    void push_back(uint8_t b) {
        if (!ext) { own.push_back(b); return; }
        if (ext_n < ext_cap) ext[ext_n++] = b; else overflow = true;
    }
    void append(const uint8_t* p, size_t n) {
        if (!ext) { own.insert(own.end(), p, p + n); return; }
        if (ext_n + n <= ext_cap) { memcpy(ext + ext_n, p, n); ext_n += n; } else overflow = true;
    }
    void swap(std::vector<uint8_t>& v) { own.swap(v); }     // storage recycling of the owned mode
};

struct Jpeg {
    // ---- read_jpeg products (jpgcoder.cc:2270-2466)
    std::vector<uint8_t> hdr;        // every marker segment after SOI, in file order ("hdrdata")
    HuffBuf huff;                    // entropy-coded bytes of all scans, de-stuffed, RST markers removed ("huffdata")
    std::vector<uint8_t> grb;        // bytes from EOI on ("grbgdata"); empty when exactly FF D9
    std::vector<uint8_t> prefix;     // -embedding=N: the N bytes in front of the JPEG's SOI ("prefix_grbgdata", 'PGE' section)
    std::vector<std::pair<uint32_t, uint32_t>> offs;   // (position in huff, position in file) ("huff_input_offsets")
    std::vector<uint32_t> rst_cnt;   // restart markers seen per scan
    std::vector<uint8_t> rst_err;    // trailing bogus restart markers per scan
    bool early_eof = false;
    uint32_t filesize = 0;           // the whole input, prefix included ("jpgfilesize")
    // ---- frame (setup_imginfo_jpg, jpgcoder.cc:4450-4540)
    int jpegtype = 0;                // 1 sequential, 2 progressive
    int width = 0, height = 0, ncmp = 0;
    Component cmp[4];
    uint16_t qtables[4][64] = {};    // zig-zag order as stored in DQT
    bool qt_set[4] = {false, false, false, false};
    int mcuh = 0, mcuv = 0, mcuc = 0;
    // ---- decode products (decode_jpeg, jpgcoder.cc:2799-3302)
    int8_t padbit = -1;
    bool is_baseline = true;         // false: progressive, or scans that do not interleave all components (flag 'X')
    int max_cmp = 0, max_bpos = 0, max_sah = 0, max_dpos[4] = {0, 0, 0, 0};   // truncation bookkeeping (EEE section)
    int trunc_bcv[4] = {0, 0, 0, 0}, trunc_bc[4] = {0, 0, 0, 0};             // coded rows / blocks per component
    std::vector<Handoff> rows;       // one per MCU row + the final one ("luma_row_offset_return")
    int status = OK;
    std::string error;
};

// Parse the container level of a JPEG file (everything except Huffman decoding).  `data` starts at SOI unless
// `embedding` >= 0 (-embedding=N, read_jpeg jpgcoder.cc:2275-2282): then the JPEG's two SOI bytes sit at byte `embedding`,
// the bytes in front of them become j.prefix, and, as in the reference, the two bytes there are skipped without a look.
// File positions (handoffs, filesize) count from the start of `data`, prefix included.  `discard_meta` (-d,
// rebuild_header_jpg :4848-4888) keeps only the header segments the coefficients need (DQT, DHT, DRI, SOF0-2, SOS).
bool parse_jpeg(const uint8_t* data, size_t n, Jpeg& j, long long embedding = -1, bool discard_meta = false);
// Frame geometry + quantisation tables from j.hdr (setup_imginfo_jpg); used by both directions.
bool parse_frame(Jpeg& j);
// Header-only peek: total (256-byte padded) bytes of all coefficient planes, 0 if unknown.  `embedding` as for parse_jpeg.
size_t peek_plane_bytes(const uint8_t* data, size_t n, long long embedding = -1);
// Bytes of coefficient plane c (AlignedBlock order).
inline size_t plane_bytes(const Jpeg& j, int c) { return (size_t)j.cmp[c].bc * 128; }
// Huffman-decode all scans into planes (pre-zeroed, AlignedBlock order) and record the per-row handoffs.
bool decode_scans(Jpeg& j, int16_t* const planes[4]);

// ---- GPU Huffman path helpers
struct GpuScanSetup {
    int rsti = 0;
    lepb200_hufftable dc[3], ac[3];  // tables selected by the SOS for each component (frame order == scan order)
};
// sos_end (optional) receives the end of the SOS segment inside j.hdr.
bool gpu_scan_setup(const Jpeg& j, GpuScanSetup& out, size_t* sos_end = nullptr);
Handoff handoff_from_state(const Jpeg& j, uint32_t bitpos, int mcu_y, const int16_t lastdc[3]);

// ---- container ----------------------------------------------------------------------------------
struct Splits {
    std::vector<Handoff> selected;   // what gets serialised into the header ('H' 'H' nseg ...)
};
// Thread-segment selection of write_ujpg (jpgcoder.cc:3860-3934) with the reference's default options.
Splits select_splits(const Jpeg& j, unsigned max_threads = 8, unsigned min_threads = 1, bool even_split = false);

// MuxWriter + vp8_full_encoder interleave schedule (src/io/MuxReader.hh:336-522, src/lepton/vp8_encoder.cc:573-600).
// One packet of the mux: `nhdr` header bytes, then `len` bytes of stream `id` from offset `src_off`.  plan_mux runs the
// writer on stream LENGTHS only (its decisions never depend on the data); mux_streams copies by the plan.
typedef lepb200_mux_packet MuxPacket;            // include/lepton_b200.h
void plan_mux(const size_t* lens, int nseg, std::vector<MuxPacket>& out);
void mux_streams(const std::vector<std::pair<const uint8_t*, size_t>>& streams, std::vector<uint8_t>& out);
// fixed header + zlib'd header blob + "CMP": everything of a .lep in front of the mux packets
bool build_lep_header(const Jpeg& j, const Splits& sp, std::vector<uint8_t>& out, std::string& err);

// Whole .lep file: fixed header, zlib'd header blob, "CMP", muxed streams, LE32 size trailer.
bool write_lep(const Jpeg& j, const Splits& sp, const std::vector<std::pair<const uint8_t*, size_t>>& streams,
               std::vector<uint8_t>& out, std::string& err);

// The generic container of -permissive (generic_compress.cc:60-200), for files the coder cannot take: flag 'Y', a fixed
// 1x1 grey JPEG header, GENERIC_SEGMENTS zeroed handoffs, the whole input in the PGE section, an empty GRB section and no
// coded streams.  Restoring it gives the input back byte for byte.  An empty input has none (false).
enum { GENERIC_SEGMENTS = 8 };                   // the reference's MAX_NUM_THREADS, whatever -maxencodethreads says
const std::vector<uint8_t>& generic_jpeg_header();   // the HDR section of every generic container
bool write_generic_lep(const uint8_t* data, size_t n, std::vector<uint8_t>& out, std::string& err);

// ---- decode side --------------------------------------------------------------------------------------
struct LepFile {
    uint8_t version = 0, flag = 0;
    int nseg = 0;
    uint32_t jpeg_size = 0;
    Jpeg j;                          // hdr, grb, rst_cnt/rst_err, padbit, frame filled from the header blob
    std::vector<Handoff> handoffs;   // as serialised (luma_y_start, segment_size, overhang, last_dc)
    bool has_eee = false;
    bool rst_cnt_set = false;        // CRS section present (jpgcoder.cc:4241)
    bool legacy = false;             // no handoff table: segment rows read from the payload (vp8_decoder.cc:337-369)
    bool zlib0 = false;              // magic CE B6 (zeta) instead of CF 84 (tau): the JPEG is handed out as a zlib stream
    bool generic = false;            // the generic container of -permissive: the file is j.prefix, nothing is coded (nseg 0)
    uint32_t eee[7] = {0};
    std::vector<std::vector<uint8_t>> streams;   // demuxed per-segment bool-coder streams
    // read_lep(..., lazy = true): the mux packets of every stream as (pointer into the caller's file, length) instead of a
    // copy -- the batch decoder gathers them straight into its pinned staging buffer; `streams` then stays empty
    std::vector<std::vector<std::pair<const uint8_t*, uint32_t>>> spans;
    std::vector<size_t> stream_len;
    size_t member_end = 0;           // bytes up to and including the mux's EOF marker; 0 without one (version 1)
    int status = OK;
    std::string error;
};
// `carry` (member walk only): in, the header sections a -lepcat file's first member left for this one (the container's own
// blob must then be empty); out, the sections behind this member's CNT marker.  Without it a CNT marker is unknown data.
bool read_lep(const uint8_t* data, size_t n, LepFile& lf, bool lazy = false, std::vector<uint8_t>* carry = nullptr);
// The members of a stream of concatenated .lep files (`cat a.lep b.lep`, -lepcat files; process_file, jpgcoder.cc:1867-1898):
// every member read_lep gives, up to and including the first that fails.  The stream ends behind a member without an EOF
// marker (version 1), or where fewer than 6 bytes follow the marker, or where the 2 bytes behind the size trailer are not
// the first member's magic.  A progressive ('X') member behind a 'Z' one fails with ASSERTION_FAILURE, as the reference's
// baseline re-encoder does on it.
void read_lep_members(const uint8_t* data, size_t n, std::vector<std::unique_ptr<LepFile>>& out, bool lazy);
bool brotli_available();          // libbrotlidec could be loaded: container versions 2 / 4 (brotli header blob) are read
// Set-up for re-encoding the scan on the GPU (lepb200_huffman_encode_resident): false when the file needs the host
// re-encoder (progressive, truncated, several scans, scan order != frame order, restart-marker budget).
struct GpuRecodeSetup : GpuScanSetup {
    size_t hpos = 0;                 // end of the first SOS segment inside hdr
    uint32_t scan_bytes = 0;         // entropy-coded bytes of the scan in the original file
};
bool gpu_recode_setup(const LepFile& lf, GpuRecodeSetup& out);
// The zlib0 stream of an n-byte payload: 78 01, stored deflate blocks of 65535 bytes (5-byte header: BFINAL, LEN, NLEN little-
// endian) of which the last one is BFINAL and never empty, then the big-endian Adler-32 -- 2 + n + 5 ceil(n / 65535) + 4 bytes.
size_t zlib0_size(size_t n);
// Frames `n` bytes in one copy into `out` (resized to zlib0_size(n)), taking their Adler-32 on the way.
void zlib0_frame(const uint8_t* data, size_t n, std::vector<uint8_t>& out);
// JPEG bytes around a scan produced elsewhere: SOI + header up to the SOS + scan + trailing restart markers + rest of the
// header + garbage (the tail of recode_baseline_jpeg, recoder.cc:839-886).  With `zlib0`, a zlib stream of stored blocks
// (-zlib0, Zlib0Writer of src/io/Zlib0.cc) whose Adler-32 combines `scan_adler`, the device's sum of the scan bytes
// (lepb200_huffman_encode_adler32), with the host's sums of the header and trailer bytes.  With `member_adler` as well
// (a member of a concatenated stream restored as one zlib stream), `out` gets the plain JPEG and *member_adler that sum.
bool assemble_baseline(const LepFile& lf, const GpuRecodeSetup& gs, const uint8_t* scan, std::vector<uint8_t>& out, std::string& err,
                       bool zlib0 = false, uint32_t scan_adler = 1, uint32_t* member_adler = nullptr);
// Re-create the JPEG bytes from decoded coefficient planes (recode_baseline_jpeg, src/lepton/recoder.cc:694-889).  A zlib0
// output is recoded into a per-thread buffer first and framed from there (the host takes the whole Adler-32).
bool recode_baseline(const LepFile& lf, const int16_t* const planes[4], std::vector<uint8_t>& out, std::string& err,
                     bool zlib0 = false, uint32_t* member_adler = nullptr);
// ONE zlib0 stream over the concatenated parts (the reference keeps one Zlib0Writer across the members of a stream,
// bounded_iostream::prep_for_new_file): blocks of 65535 bytes run across part borders, and the Adler-32 is combined from
// the parts' sums.
void zlib0_join(const std::vector<std::pair<const uint8_t*, size_t>>& parts, const uint32_t* adlers, std::vector<uint8_t>& out);

}  // namespace lephost
