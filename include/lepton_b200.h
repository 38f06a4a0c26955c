/*
 * lepton_b200.h -- C ABI of the CUDA Lepton arithmetic-coding path (sm_90a).
 *
 * This is the drop-in boundary for the reference's BaseEncoder / BaseDecoder plug-in interface
 * (/root/reference/src/lepton/base_coders.hh:26-65):
 *
 *   lepb200_encode_images  replaces  BaseEncoder::encode_chunk(const UncompressedComponents*, FileWriter*,
 *                                    const ThreadHandoff* selected_splits, unsigned num_selected_splits)
 *                          (base_coders.hh:59-62, called from write_ujpg, src/lepton/jpgcoder.cc:4079-4081),
 *                          i.e. VP8ComponentEncoder::vp8_full_encoder up to -- not including -- the MuxWriter
 *                          interleave (src/lepton/vp8_encoder.cc:521-573): it returns one bool-coder byte
 *                          stream per thread-segment.  Batched over images.
 *   lepb200_decode_images  replaces  BaseDecoder::decode_chunk(UncompressedComponents*) /
 *                          BaseDecoder::decode_row (base_coders.hh:31,38-44; src/lepton/vp8_decoder.cc:387-490,
 *                          src/lepton/lepton_codec.cc:266-309): demuxed per-segment streams in, full
 *                          coefficient planes out.
 *
 * Plain pointers and sizes only; no C++/torch types.  All hot-path compute runs in hand-written sm_90a
 * CUDA kernels; there is no CPU fallback: without a CUDA device every entry point that needs one fails
 * with LEPB200_ERR_NO_DEVICE.
 *
 * Data layout at the boundary is the reference's: a component plane is a row-major array of AlignedBlock
 * (64 x int16, 128 bytes; order: 49 "7x7" coefficients in zig-zag order, DC, 7 row-0 ACs, 7 column-0 ACs;
 * src/vp8/util/aligned_block.hh:32-44,98-161), `bch` blocks per row, `bcv` rows
 * (src/lepton/uncompressed_components.hh:24-302).
 */
#ifndef LEPTON_B200_H_
#define LEPTON_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LEPB200_MAX_SEGMENTS 16 /* MuxReader::MAX_STREAM_ID, src/io/MuxReader.hh:201 */

/* return codes of the API itself (per-segment coding status uses the reference's ExitCode values) */
enum {
    LEPB200_OK = 0,
    LEPB200_ERR_NO_DEVICE = -1,
    LEPB200_ERR_CUDA = -2,
    LEPB200_ERR_INVALID = -3,
    LEPB200_ERR_NOMEM = -4
};

/* per-segment status: reference ExitCode values (src/vp8/util/memory.hh:13-39) */
enum {
    LEPB200_ST_SUCCESS = 0,
    LEPB200_ST_ASSERTION_FAILURE = 1,
    LEPB200_ST_COEFFICIENT_OUT_OF_RANGE = 6,
    LEPB200_ST_STREAM_INCONSISTENT = 7,
    LEPB200_ST_UNSUPPORTED_JPEG_WITH_ZERO_IDCT_0 = 43,
    LEPB200_ST_OUTPUT_OVERFLOW = 100 /* not a reference code: the caller-independent output arena was too small */
};

typedef struct lepb200_ctx lepb200_ctx;

/* One image = what UncompressedComponents + the selected ThreadHandoff splits carry across the boundary. */
typedef struct lepb200_image {
    int32_t ncmp;                    /* 1..3 colour components (get_num_components) */
    int32_t mcuv;                    /* MCU rows (get_mcu_count_vertical) */
    int32_t bch[3];                  /* blocks per row of each component plane (block_width) */
    int32_t bcv[3];                  /* allocated block rows (original_height) */
    int32_t trunc_bcv[3];            /* rows actually coded (get_max_coded_heights); == bcv unless truncated */
    int32_t trunc_bc[3];             /* blocks actually coded (component_size_in_blocks); == bch*bcv unless truncated */
    uint16_t qtable_zigzag[3][64];   /* get_quantization_tables(cmp): DQT entries in zig-zag order */
    int16_t* planes[3];              /* HOST memory, bch*bcv AlignedBlocks each; input for encode, output for decode */
    int32_t nseg;                    /* number of thread-segments, 1..16 (selected_splits) */
    int32_t luma_y_start[LEPB200_MAX_SEGMENTS]; /* ThreadHandoff::luma_y_start of each segment; segment i ends
                                                    where i+1 starts, the last one runs to the end of the image */
    uint32_t seg_token_bound[LEPB200_MAX_SEGMENTS]; /* encode, optional: upper bound of the binary decisions of each segment
                                                    (from lepb200_huffrow.tokens); 0 = unknown, the library counts itself */
} lepb200_image;

/* One thread-segment's bool-coder stream. */
typedef struct lepb200_stream {
    const uint8_t* data;             /* encode: points into memory owned by the context, valid until the next call */
    uint64_t len;
    int32_t status;                  /* LEPB200_ST_* */
    uint32_t reserved;
    uint64_t ndecisions;             /* binary decisions coded (VPXBoolWriter::put / VPXBoolReader::get calls) */
} lepb200_stream;

/* Creates a context on CUDA device `device` (one context per GPU / per host thread). */
int lepb200_create(lepb200_ctx** out, int device);
void lepb200_destroy(lepb200_ctx* ctx);
/* Frees the context's device arenas (they grow again on the next call); the context stays usable. */
void lepb200_release_device_buffers(lepb200_ctx* ctx);
const char* lepb200_last_error(const lepb200_ctx* ctx);

/* Page-locked host memory for planes / streams handed to the calls below (pageable memory works too, slower). */
void* lepb200_pinned_alloc(size_t bytes);
void lepb200_pinned_free(void* p);

/* ---- one-call forms (host buffers in, host buffers out; H2D + kernel + D2H) ---- */
/* out must have room for sum(images[i].nseg) entries, filled image-major. */
int lepb200_encode_images(lepb200_ctx* ctx, const lepb200_image* images, int nimages, lepb200_stream* out);
/* in has sum(images[i].nseg) entries (data/len used); decoded planes are written to images[i].planes.
 * status_out (optional) receives one LEPB200_ST_* per segment. */
int lepb200_decode_images(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const lepb200_stream* in,
                          int32_t* status_out);

/* ---- staged forms (for pipelining and for timing the kernel with inputs resident in HBM) ---- */
int lepb200_encode_upload(lepb200_ctx* ctx, const lepb200_image* images, int nimages); /* H2D planes + job tables */
int lepb200_encode_launch(lepb200_ctx* ctx);                                           /* kernel only (async) */
/* the two halves of lepb200_encode_launch, for callers that pipeline them over different batches: symbolisation +
 * model update (the heavy, throughput-bound kernel) and the serial range-coder chains (latency-bound, a few warps) */
int lepb200_encode_launch_symbolise(lepb200_ctx* ctx);
int lepb200_encode_launch_rangecode(lepb200_ctx* ctx);
int lepb200_encode_fetch(lepb200_ctx* ctx, lepb200_stream* out);                       /* sync + D2H streams */
/* Test entry: an encode batch from caller token streams instead of kernel A, ready for lepb200_encode_launch_rangecode
 * and lepb200_encode_fetch / lepb200_encode_fetch_files.  Segment s has ntok[s] tokens (probability | bit << 8; all
 * segments back to back in `tokens`) and a stream slot of caps[s] bytes; the segments form nfiles files of seg_per_file[f]
 * consecutive segments each.  The stream arena and the overflow arena of the batch are filled with canary bytes. */
int lepb200_encode_upload_tokens(lepb200_ctx* ctx, const uint16_t* tokens, const uint32_t* ntok, const uint32_t* caps, int nseg,
                                 const int32_t* seg_per_file, int nfiles);
/* After the fetch of such a batch: moved[s] = 1 where stream s was placed in the overflow arena (it did not fit its slot),
 * *changed = canary bytes overwritten behind the slots and behind the streams of the overflow arena. */
int lepb200_encode_token_canaries(lepb200_ctx* ctx, uint8_t* moved, uint64_t* changed);
/* lepb200_encode_upload_tokens with the entropy coder of every segment: coders[s] (LEPB200_CODER_*) for segment s, NULL = all
 * LEPB200_CODER_BOOL (then exactly lepb200_encode_upload_tokens).  lepb200_encode_launch_rangecode codes the rANS segments
 * with the rANS pass: their streams are written into their token slots, so caps[s] does not matter for them and
 * lepb200_encode_token_canaries reports them as moved.  Fetch with lepb200_encode_fetch. */
int lepb200_encode_upload_tokens_coded(lepb200_ctx* ctx, const uint16_t* tokens, const uint32_t* ntok, const uint32_t* caps, int nseg,
                                       const int32_t* seg_per_file, int nfiles, const uint8_t* coders);
int lepb200_decode_upload(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const lepb200_stream* in);
int lepb200_decode_launch(lepb200_ctx* ctx);
int lepb200_decode_fetch(lepb200_ctx* ctx, const lepb200_image* images, int nimages, int32_t* status_out);
/* Per-segment decision counts of the batch the last lepb200_decode_fetch returned (out: one per segment, in batch order):
 * the decisions each segment's decode took before it ended, well or not.  LEPB200_ERR_INVALID before that fetch. */
int lepb200_decode_fetch_decisions(lepb200_ctx* ctx, uint64_t* out);

/* Wait for everything queued on the context's stream. */
int lepb200_sync(lepb200_ctx* ctx);
/* ---- GPU Huffman decode (SURVEY.md 8(f) row 1): baseline JPEG scan -> coefficient planes directly in HBM.
 * Replaces the Huffman half of decode_jpeg (src/lepton/jpgcoder.cc:2799-3302, decode_block_seq :4893-4961); the caller
 * still parses markers and de-stuffs the entropy-coded bytes (read_jpeg, :2270-2466).  One thread per image. */
typedef struct lepb200_hufftable { uint8_t bits[17]; uint8_t vals[256]; } lepb200_hufftable;   /* DHT form: counts per length (bits[1..16]) + symbols */
typedef struct lepb200_huffrow { uint32_t bitpos; int16_t lastdc[3]; int16_t mcu_y; uint32_t tokens; } lepb200_huffrow; /* Huffman state at an MCU-row start;
   tokens = upper bound of the coder's binary decisions for all blocks before the row */
typedef struct lepb200_jpeg_scan {
    const uint8_t* entropy;          /* HOST: de-stuffed entropy-coded bytes of the (single) scan, RST markers removed.
                                      * NULL = placeholder: the image only gets its (zeroed) plane slot in the device arena and is
                                      * filled from host planes by lepb200_encode_upload_resident (files the host had to decode) */
    uint32_t nbytes;
    int32_t ncmp, mcuh, mcuv, rsti;  /* components (frame order == scan order), MCUs per row / rows, restart interval */
    int32_t H[3], V[3];              /* sampling factors */
    int32_t nch[3], ncv[3];          /* non-interleaved block counts (single-component scans) */
    lepb200_hufftable dc[3], ac[3];  /* tables selected by the SOS for each component */
    /* outputs */
    int32_t status;                  /* 0 ok, 42 UNSUPPORTED_JPEG (decode error, inconsistent padding, trailing data), 200 not handled */
    int32_t padbit;                  /* as written to the P0D section */
    uint32_t end_bitpos;
    int32_t nrows;
    lepb200_huffrow* rows;           /* HOST array with room for mcuv + 1 entries */
} lepb200_jpeg_scan;
/* Uploads the entropy bytes, Huffman-decodes every scan into the context's device plane arena (laid out exactly as a
 * following lepb200_encode_upload_resident expects) and returns per-row states + status on the host. */
int lepb200_huffman_decode_to_device(lepb200_ctx* ctx, lepb200_jpeg_scan* scans, int nimages);
/* Pinned staging buffer of the context (>= bytes): scans whose `entropy` pointers lie inside it, 16-byte aligned and with
 * >= 16 spare bytes behind each, are uploaded by lepb200_huffman_decode_to_device without the gather copy. */
uint8_t* lepb200_huffman_stage_reserve(lepb200_ctx* ctx, size_t bytes);
/* Optional: push staged bytes [offset, offset + bytes) to the device right away (asynchronous, thread-safe), e.g. from the
 * thread that just parsed a file, so that the H2D copy overlaps the parsing of the other files.  The caller then uploads
 * EVERY scan of the batch this way (with the 16 bytes behind each scan zeroed). */
int lepb200_huffman_stage_upload(lepb200_ctx* ctx, size_t offset, size_t bytes);
/* Like lepb200_encode_upload, but the planes are the ones just produced on the device by
 * lepb200_huffman_decode_to_device (geometry must match scan i).  images[i].planes == NULL: use the resident planes;
 * non-NULL (placeholder scans): copy these host planes into the image's slot first. */
int lepb200_encode_upload_resident(lepb200_ctx* ctx, const lepb200_image* images, int nimages);

/* ---- GPU baseline Huffman ENCODE for the decode direction (SURVEY 8(f) row 2; reference: recode_row_range /
 * recode_one_mcu_row / encode_block_seq / escape_0xff_huffman_and_write, src/lepton/recoder.cc:472-545,316-410,245-313,
 * 144-185).  After lepb200_decode_launch on the same context, image i of the batch (single interleaved or grey baseline
 * scan, not truncated) gets the entropy-coded bytes of its scan -- stuffed, with restart markers -- produced on the
 * device from the resident planes, one warp per thread-segment, so the D2H copy carries JPEG bytes, not 128 B per block.
 * scan_bytes == 0 skips an image (the caller re-encodes it on the host from the fetched planes). */
typedef struct lepb200_henc_segment {
    int32_t mcu_row_start, mcu_row_end;   /* MCU rows [start, end) of the thread-segment */
    int16_t last_dc[3];                   /* ThreadHandoff::last_dc */
    uint8_t overhang_bits, overhang_byte; /* ThreadHandoff::num_overhang_bits / overhang_byte */
    uint32_t expect_bytes;                /* ThreadHandoff::segment_size (file bytes the segment covers); ignored for the last one */
} lepb200_henc_segment;
typedef struct lepb200_henc_image {
    int32_t rsti, padbit;
    int32_t H[3], V[3];                   /* sampling factors (frame order == scan order) */
    lepb200_hufftable dc[3], ac[3];       /* tables selected by the SOS for each component */
    int32_t nseg;
    lepb200_henc_segment seg[LEPB200_MAX_SEGMENTS];
    uint32_t scan_bytes;                  /* bytes the scan must produce (file size - markers - trailer); 0 = skip this image */
    /* outputs of lepb200_huffman_encode_fetch */
    const uint8_t* data;                  /* HOST (pinned, owned by the context): scan_bytes bytes */
    int32_t status;                       /* 0 ok; 1 a segment did not produce the byte count its handoff promises */
} lepb200_henc_image;
int lepb200_huffman_encode_resident(lepb200_ctx* ctx, lepb200_henc_image* images, int nimages);   /* queues the kernel (async) */
int lepb200_huffman_encode_fetch(lepb200_ctx* ctx, lepb200_henc_image* images, int nimages);      /* waits, D2H of the scan bytes */
/* The same in `nparts` launches over consecutive images (about equal output bytes each), every launch followed by the D2H
 * of its scan bytes on a second stream: part k travels, and the caller assembles its files, while part k + 1 is encoded.
 * lepb200_huffman_encode_parts = parts actually queued; lepb200_huffman_encode_wait_part blocks until part `part` is on the
 * host, fills data / status of its images and returns their index range [*first, *last). */
int lepb200_huffman_encode_resident_parts(lepb200_ctx* ctx, lepb200_henc_image* images, int nimages, int nparts);
int lepb200_huffman_encode_parts(const lepb200_ctx* ctx);
int lepb200_huffman_encode_wait_part(lepb200_ctx* ctx, lepb200_henc_image* images, int nimages, int part, int* first, int* last);
/* Adler-32 (RFC 1950) of the scan bytes of images [first, last) of the batch, taken by the encode kernel while it wrote them
 * (each warp over its thread-segment; the segments are combined here in order): adler[i] for i in [first, last).  Valid for
 * images whose part lepb200_huffman_encode_wait_part returned, or after lepb200_huffman_encode_fetch; meaningful where the
 * image's status is 0.  A skipped image (scan_bytes == 0) gets 1, the Adler-32 of no bytes. */
int lepb200_huffman_encode_adler32(lepb200_ctx* ctx, int first, int last, uint32_t* adler);
/* Per-segment status of the decode batch as soon as the decode kernel has finished (a second stream: work queued behind
 * the kernel -- the Huffman encode above -- is not waited for).  lepb200_decode_fetch reports the same later. */
int lepb200_decode_fetch_status(lepb200_ctx* ctx, int32_t* status_out);

/* Device time of the most recent *_launch (CUDA events on the context's stream), milliseconds; <0 if none. */
float lepb200_last_kernel_ms(lepb200_ctx* ctx);
/* Encode only: device time of kernel A (symbolisation + model update) within the last launch; the rest of
 * lepb200_last_kernel_ms is kernel B (range coder). */
float lepb200_last_symbolise_ms(lepb200_ctx* ctx);
/* Device time of the Huffman-decode kernel of the last lepb200_huffman_decode_to_device call, milliseconds. */
float lepb200_last_huffman_ms(lepb200_ctx* ctx);
/* Synchronisation iterations the sub-sequence Huffman kernels (lep_huffpar.cu) needed in that call; 0 = serial kernel only. */
int lepb200_last_huffman_iterations(lepb200_ctx* ctx);
/* Images of that call the sub-sequence kernels did not finish cleanly (an anomaly, or no convergence within the iteration
 * budget), so that the serial kernel decoded them again from the start. */
int lepb200_last_huffman_redone(lepb200_ctx* ctx);
/* Number of kernel launches issued by this context so far (for bench.py's gpu_launches). */
uint64_t lepb200_kernel_launches(const lepb200_ctx* ctx);
/* Sum over the last uploaded batch of 128 * coded blocks + stream bytes (SURVEY.md section 8(d) algorithmic bytes);
 * valid after *_fetch. */
uint64_t lepb200_last_algorithmic_bytes(const lepb200_ctx* ctx);
/* Size in bytes of one per-warp probability model (informational). */
size_t lepb200_model_bytes(void);
/* Co-scheduling knobs (no reference counterpart): cap the persistent encode grid at n CTAs per SM (0 = fill the SM) and
 * set how many images one CTA of the Huffman kernel decodes, so that the Huffman decode of the next chunk runs NEXT TO
 * the encode kernel of the current one instead of behind it.  Environment LEPB200_ENC_CTA_CAP / LEPB200_HUFF_WARPS override. */
void lepb200_set_encode_ctas_per_sm(lepb200_ctx* ctx, int n);
void lepb200_set_host_threads(lepb200_ctx* ctx, int n);   /* host threads the context may use for staging copies (default 1) */
void lepb200_set_huffman_warps_per_cta(lepb200_ctx* ctx, int n);
/* 1 if a CUDA device is usable from this process. */
int lepb200_device_available(void);


/* ------------------------------------------------------------------------------------------------------------
 * File-level drop-in (host front/back end + GPU coder): what `lepton in.jpg out.lep` / `lepton in.lep out.jpg`
 * do (src/lepton/jpgcoder.cc process_file :1528), batched over files.  Outputs are byte-identical to the
 * reference CLI with default options.  status is a reference ExitCode (0 ok) or LEPB200_ST_NOT_HANDLED for
 * inputs whose host-side handling this build does not cover yet (such files are refused, never mis-coded).
 * ------------------------------------------------------------------------------------------------------------ */
#define LEPB200_ST_NOT_HANDLED 200

typedef struct lepb200_codec lepb200_codec;
typedef struct lepb200_buffer { const uint8_t* data; size_t len; } lepb200_buffer;
typedef struct lepb200_result { const uint8_t* data; size_t len; int32_t status; } lepb200_result; /* data owned by the codec */
/* lepb200_decode_upload for streams that lie in pieces (the mux packets of a .lep file, src/io/MuxReader.hh:230-283): in[s].len
 * is the length of segment s's stream, its bytes are the pieces spans[span_first[s] .. span_first[s + 1]) in order; in[s].data
 * is not read.  The pieces are gathered straight into the context's pinned staging buffer (no intermediate copy). */
/* Instead of lepb200_encode_fetch: one complete .lep file per image of the batch, ASSEMBLED ON THE DEVICE.  headers[i] =
 * everything in front of the mux packets (fixed header, compressed JPEG header, "CMP" -- jpgcoder.cc:3779-4076; the host
 * stages build it, lepb200_host_jpeg_header); the MuxWriter packet schedule (src/io/MuxReader.hh:336-522) is planned
 * from the stream lengths and a gather kernel writes header, packets and the LE32 size trailer (vp8_encoder.cc:573-614) into
 * one dense buffer that comes back in a single copy.  files[i].data: pinned host memory owned by the context (valid until its
 * next fetch); files[i].status: the first non-zero segment status of the image (then no file). */
int lepb200_encode_fetch_files(lepb200_ctx* ctx, const lepb200_buffer* headers, lepb200_result* files);
int lepb200_decode_upload_gather(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const lepb200_stream* in,
                                 const lepb200_buffer* spans, const uint32_t* span_first);
/* Entropy coder of an image's segment streams.  LEPB200_CODER_BOOL: the VP8 bool coder of .lep container versions 1, 2 and 4,
 * what every decode entry point without a coder argument reads.  LEPB200_CODER_ANS: the two-state rANS coder of container
 * version 3 (the reference's -ans option, src/vp8/decoder/ans_bool_reader.hh): the same grammar and model layout, its own
 * update of the branch counts (Branch::adv_record_obs_and_update) and other bits. */
#define LEPB200_CODER_BOOL 0
#define LEPB200_CODER_ANS 1
/* lepb200_encode_upload / lepb200_encode_images with the coder of every image: coders[i] (LEPB200_CODER_*) for image i,
 * NULL = all LEPB200_CODER_BOOL (then exactly the forms without it).  A batch may mix coders: kernel A runs once per coder,
 * the bool coder's range coder codes the bool-coded segments and the rANS pass the rANS-coded ones (container version 3,
 * the reference's -ans).  The streams come back through lepb200_encode_fetch in the caller's order;
 * lepb200_encode_fetch_files refuses a batch with rANS-coded segments (LEPB200_ERR_INVALID): it writes version-1 files only. */
int lepb200_encode_upload_coded(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const uint8_t* coders);
int lepb200_encode_images_coded(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const uint8_t* coders, lepb200_stream* out);
/* lepb200_decode_upload / lepb200_decode_upload_gather with the coder of every image: coders[i] (LEPB200_CODER_*) for image i,
 * NULL = all LEPB200_CODER_BOOL (then exactly the forms without it).  A batch may mix coders: the segments of each coder are
 * decoded by launches of their own, each choosing its kernel by its own size.  Launch and fetch as for the plain forms. */
int lepb200_decode_upload_coded(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const lepb200_stream* in,
                                const uint8_t* coders);
int lepb200_decode_upload_gather_coded(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const lepb200_stream* in,
                                       const lepb200_buffer* spans, const uint32_t* span_first, const uint8_t* coders);

int lepb200_codec_create(lepb200_codec** out, int device, int host_threads /* 0 = all cores */);
void lepb200_codec_destroy(lepb200_codec* codec);
const char* lepb200_codec_last_error(const lepb200_codec* codec);
lepb200_ctx* lepb200_codec_ctx(lepb200_codec* codec);
/* kernel launches issued so far by the codec's contexts */
uint64_t lepb200_codec_kernel_launches(const lepb200_codec* codec);
/* files per pipeline chunk (default 1024): chunk k+1 is Huffman-decoded while chunk k is on the GPU */
void lepb200_codec_set_chunk_images(lepb200_codec* codec, int n);
/* 1 (default): Huffman-decode on the GPU when every file of a chunk is a complete single-scan baseline JPEG;
 * 0: always Huffman-decode on host threads */
void lepb200_codec_set_gpu_huffman(lepb200_codec* codec, int on);
/* 1 (default, the reference built with DEFAULT_ALLOW_PROGRESSIVE / run with -allowprogressive): progressive and
 * non-interleaved JPEGs are coded; 0 (-rejectprogressive): they fail with the reference's exit code 8
 * (PROGRESSIVE_UNSUPPORTED, src/lepton/jpgcoder.cc:2911-2925) */
void lepb200_codec_set_allow_progressive(lepb200_codec* codec, int on);
/* -minencodethreads=N / -maxencodethreads=N of the reference CLI (src/lepton/jpgcoder.cc:1080-1089): bounds of the
 * thread-segment count write_ujpg selects (:3862-3874); both clamp to 1..8, defaults 1 and 8.  They change the .lep
 * bytes exactly as they do in the reference. */
void lepb200_codec_set_encode_threads(lepb200_codec* codec, int min_threads, int max_threads);
/* -verify / -roundtrip of the reference CLI (its default; src/lepton/jpgcoder.cc:1095-1110, validation.cc): 1 = every
 * .lep produced by lepb200_compress_jpegs is decoded again on the GPU and compared with the input; a file that does not
 * come back byte for byte is withheld with status 41 (ROUNDTRIP_FAILURE), e.g. the reference's images/roundtripfail.jpg.
 * 0 (default) = -skipverify. */
void lepb200_codec_set_verify(lepb200_codec* codec, int on);
/* -evensplit (jpgcoder.cc:1063-1064, :3898-3900): thread-segments cover equal numbers of MCU rows instead of equal bytes */
void lepb200_codec_set_even_split(lepb200_codec* codec, int on);
/* -zlib0 (jpgcoder.cc:2089, check_file :2200-2220, src/io/Zlib0.cc): 1 = lepb200_decompress_leps hands every restored JPEG out
 * as a zlib stream: 78 01, stored deflate blocks of 65535 bytes (the last one BFINAL and never empty), the big-endian Adler-32
 * of the JPEG -- 2 + n + 5 ceil(n / 65535) + 4 bytes for an n-byte JPEG.  Files whose magic is CE B6 (zeta) instead of CF 84
 * are always handed out so, whatever this setting.  The Adler-32 of a scan the device re-encodes is taken by the encode kernel,
 * that of a scan the host re-encodes by the host.  Statuses do not change; lepb200_compress_jpegs
 * ignores the setting, as the reference does.  0 (default): plain JPEG bytes. */
void lepb200_codec_set_zlib0(lepb200_codec* codec, int on);
/* -embedding=N (jpgcoder.cc:1135-1137, read_jpeg :2275-2282): offset >= 0 makes lepb200_compress_jpegs take every input as a
 * JPEG whose SOI sits at byte `offset` of a larger file.  The bytes in front of it go to the container's PGE section and
 * are written back in front of the SOI on restore, bytes after the EOI to its GRB section as always; the coded JPEG takes
 * the same device path as a plain one.  As in the reference, the two bytes at `offset` are not looked at, an offset past
 * the end of the input is ASSERTION_FAILURE (1), and 0 gives the plain .lep.  Negative (default): inputs start at their SOI. */
void lepb200_codec_set_embedding(lepb200_codec* codec, long long offset);
/* -d (rebuild_header_jpg, jpgcoder.cc:3797-3800, 4848-4888): 1 = the container keeps only the header segments the
 * coefficients are coded with (DQT, DHT, DRI, SOF0-2, SOS); APPn, COM and the rest are dropped, so the restored JPEG is
 * shorter than the input (with verification on, such a file fails with 41 as in the reference).  0 (default): all kept. */
void lepb200_codec_set_discard_meta(lepb200_codec* codec, int on);
/* -permissive (jpgcoder.cc:1111, validation.cc:25-218, generic_compress.cc:60-200): 1 = lepb200_compress_jpegs verifies every
 * file (whatever lepb200_codec_set_verify says) and stores each one that ends with a non-zero status -- not a JPEG, damaged,
 * arithmetic-coded, refused by the front end, failing verification (41), a .lep itself, inputs shorter than 2 bytes -- whole
 * in the reference's generic container instead: flag 'Y', a fixed 1x1 grey JPEG header, the input in the PGE section, no
 * coded streams.  Such a file gets status 0 and its container; only an empty input keeps a status (42, UNSUPPORTED_JPEG).
 * The other files of the call take the device path and give the bytes they give without the setting.  With -embedding or
 * -d the rule is the same, as in the reference: a -d file whose restore differs from the input fails verification and is
 * stored generically.  lepb200_decompress_leps restores generic containers (plainly or as zlib0) from their PGE section,
 * without device work; other 'Y' containers (-startbyte slices) stay refused with 200.  0 (default): off. */
void lepb200_codec_set_permissive(lepb200_codec* codec, int on);
/* device milliseconds of the last chunk's GPU Huffman-decode kernel (diagnostic) */
double lepb200_codec_last_huffman_ms(const lepb200_codec* codec);
/* files of the last lepb200_decompress_leps call whose scan was Huffman-encoded on the device (the rest went through the host re-encoder) */
int lepb200_codec_last_gpu_recoded(const lepb200_codec* codec);
/* summed seconds spent by the last call's stages (they overlap): JPEG parse + Huffman decode | H2D + kernel + D2H | container writing */
void lepb200_codec_last_timing(const lepb200_codec* codec, double* front_s, double* gpu_s, double* back_s);
/* n JPEG files in, n .lep files out */
int lepb200_compress_jpegs(lepb200_codec* codec, const lepb200_buffer* jpegs, int n, lepb200_result* out);
/* n .lep files in, n JPEG files out (byte-identical to the originals).  An input may be a stream of concatenated .lep files
 * (`cat a.lep b.lep`, -lepcat files): out[i] is then the concatenation of its members' JPEGs -- for zlib0 output ONE zlib
 * stream over all of them, as the reference writes -- and every member is one image of the call's batches.  The status of
 * such an input is that of its first member that fails; then it gets no data (the reference has written the members in
 * front of it by then). */
int lepb200_decompress_leps(lepb200_codec* codec, const lepb200_buffer* leps, int n, lepb200_result* out);

/* ---- several GPUs from one process: codecs[k] was created on its own device.  The files are dealt to the codecs
 * longest-first by size (lepb200_shard_by_size: owner[i] = codec of file i, balanced by bytes to within one file), each
 * codec codes its share through its own pipeline on its own host thread; nothing crosses between GPUs (SURVEY.md 8(e)).
 * out[i].data is owned by the codec that coded file i and stays valid until that codec's next call. */
void lepb200_shard_by_size(const size_t* sizes, int n, int world, int* owner);
int lepb200_compress_jpegs_multi(lepb200_codec* const* codecs, int ncodecs, const lepb200_buffer* jpegs, int n, lepb200_result* out);
int lepb200_decompress_leps_multi(lepb200_codec* const* codecs, int ncodecs, const lepb200_buffer* leps, int n, lepb200_result* out);

/* ---- the host stages on their own (no GPU): JPEG front end and .lep assembly around an external coder.
 * lepb200_host_jpeg_open parses + Huffman-decodes one JPEG (read_jpeg + decode_jpeg, jpgcoder.cc:2270,2799) and
 * selects the thread-segments (write_ujpg :3860-3934); *_image exposes planes/geometry/splits as a lepb200_image
 * (pointers stay valid until *_close); *_write_lep assembles the container around nseg coded streams. */
typedef struct lepb200_jpeg lepb200_jpeg;
int lepb200_host_jpeg_open(const uint8_t* data, size_t len, lepb200_jpeg** out, int32_t* status);
int lepb200_host_jpeg_open_threads(const uint8_t* data, size_t len, int min_threads, int max_threads, lepb200_jpeg** out, int32_t* status);
int lepb200_host_jpeg_open_split(const uint8_t* data, size_t len, int min_threads, int max_threads, int even_split, lepb200_jpeg** out, int32_t* status);
/* ... with -embedding=N (embedding >= 0; negative: none) and -d (discard_meta = 1), as lepb200_codec_set_embedding /
 * lepb200_codec_set_discard_meta */
int lepb200_host_jpeg_open_embedded(const uint8_t* data, size_t len, int min_threads, int max_threads, int even_split,
                                    long long embedding, int discard_meta, lepb200_jpeg** out, int32_t* status);
const char* lepb200_host_jpeg_error(const lepb200_jpeg* h);
int lepb200_host_jpeg_image(lepb200_jpeg* h, lepb200_image* img);
/* the scan as lepb200_huffman_decode_to_device takes it (de-stuffed entropy bytes, tables, geometry; pointers valid until
 * *_close; `rows` and the outputs are left alone), also when the host Huffman decoder refused the scan, as the file API
 * hands it to the device before any host decode; LEPB200_ERR_INVALID when the file needs the host Huffman decoder */
int lepb200_host_jpeg_scan(lepb200_jpeg* h, lepb200_jpeg_scan* scan);
int lepb200_host_jpeg_write_lep(lepb200_jpeg* h, const lepb200_stream* streams, int nseg, const uint8_t** data, size_t* len);
/* everything of the .lep in front of the mux packets (what lepb200_encode_fetch_files wants as headers[i]) */
int lepb200_host_jpeg_header(lepb200_jpeg* h, const uint8_t** data, size_t* len);
/* The MuxWriter schedule (src/io/MuxReader.hh:336-522 driven by vp8_encoder.cc:575-594) for nseg streams of the given
 * lengths -- it depends on the lengths only: packet k = `nhdr` header bytes, then `len` bytes of stream `id` from offset
 * `src_off`.  Returns the number of packets (writes at most `cap` of them). */
typedef struct lepb200_mux_packet { uint8_t id, nhdr, hdr[3]; uint32_t src_off, len; } lepb200_mux_packet;
int lepb200_host_mux_plan(const size_t* lens, int nseg, lepb200_mux_packet* out, int cap);
void lepb200_host_jpeg_close(lepb200_jpeg* h);
/* decode-side host stages: container parse + demux (read_ujpg, jpgcoder.cc:4117), geometry/splits, segment streams, and
 * JPEG re-creation from caller-provided planes (recode_baseline_jpeg, recoder.cc:694) */
typedef struct lepb200_lep lepb200_lep;
int lepb200_host_lep_open(const uint8_t* data, size_t len, lepb200_lep** out, int32_t* status);
const char* lepb200_host_lep_error(const lepb200_lep* h);
int lepb200_host_lep_image(lepb200_lep* h, lepb200_image* img);
int lepb200_host_lep_stream(lepb200_lep* h, int seg, const uint8_t** data, size_t* len);
int lepb200_host_lep_recode(lepb200_lep* h, const int16_t* const planes[3], const uint8_t** data, size_t* len);
/* host half of the device re-encode path (lepb200_huffman_encode_resident): offset and length of the scan in the original
 * file (both 0 when the file needs the host re-encoder), and the JPEG assembled around scan bytes produced elsewhere */
int lepb200_host_lep_scan_layout(lepb200_lep* h, uint32_t* scan_offset, uint32_t* scan_bytes);
/* 1 when the system's libbrotlidec could be loaded: .lep container versions 2, 3 and 4 (brotli-coded header blob, jpgcoder.cc:4168-4175)
 * are then read like version 1; 0: they are refused with status 200.  A version-3 file whose header blob does not brotli-decode
 * is refused with 200 as well. */
int lepb200_host_brotli_available(void);
/* LEPB200_CODER_ANS when the streams of the container opened with lepb200_host_lep_open are rANS-coded (version 3), else
 * LEPB200_CODER_BOOL: the coder argument of lepb200_decode_upload_coded for its image */
int lepb200_host_lep_coder(const lepb200_lep* h);
/* test hook: 0 when the container reader's two modes (streams copied out / mux packets recorded in place) agree on this file */
int lepb200_host_lep_lazy_equal(const uint8_t* data, size_t len);
/* the job lepb200_huffman_encode_resident wants for this file (scan_bytes == 0: the file needs the host re-encoder) */
int lepb200_host_lep_henc_image(lepb200_lep* h, lepb200_henc_image* out);
int lepb200_host_lep_assemble(lepb200_lep* h, const uint8_t* scan, size_t scan_len, const uint8_t** data, size_t* len);
void lepb200_host_lep_close(lepb200_lep* h);
/* 1 when the container opened with lepb200_host_lep_open carries the zeta magic CE B6 (its JPEG is restored as a zlib stream) */
int lepb200_host_lep_zlib0(const lepb200_lep* h);
/* Streams of concatenated .lep files (`cat a.lep b.lep`, the reference's -lepcat files; process_file, jpgcoder.cc:1867-1898):
 * lepb200_decompress_leps restores every member of every input as one image of its batch.  lepb200_host_lep_members lists the
 * members of `data` as that walk finds them: returns their number and writes up to `cap` entries.  The walk stops at the
 * first member that fails (its status is non-zero); a stream ends behind a member without an EOF marker (container version
 * 1), where fewer than 6 bytes follow the marker, or where the 2 bytes behind the member's 4-byte size trailer are not the
 * first member's magic.  lepb200_host_lep_open_member opens member `index` like lepb200_host_lep_open opens a file. */
typedef struct {
    int32_t status;          /* 0, or the reference ExitCode the member fails with */
    uint32_t jpeg_size;      /* size of the member's JPEG as its container records it */
    int32_t nseg;            /* thread-segments */
} lepb200_lep_member;
int lepb200_host_lep_members(const uint8_t* data, size_t len, lepb200_lep_member* out, int cap);
int lepb200_host_lep_open_member(const uint8_t* data, size_t len, int index, lepb200_lep** out, int32_t* status);
/* test hook: the zlib stream lepb200_codec_set_zlib0 hands out for the `len` bytes at `data`.  Returns its length; writes it
 * to `out` only when cap is at least that length. */
size_t lepb200_host_zlib0_frame(const uint8_t* data, size_t len, uint8_t* out, size_t cap);
/* host halves of -permissive: the generic container lepb200_compress_jpegs writes for the `len` bytes at `data` (returns its
 * length, 0 for an empty input; writes it to `out` only when cap is at least that length), and the bytes a generic container
 * opened with lepb200_host_lep_open restores to, as zlib0 when `zlib0` is set or the file has the zeta magic
 * (LEPB200_ERR_INVALID for any other container) */
size_t lepb200_host_generic_lep(const uint8_t* data, size_t len, uint8_t* out, size_t cap);
int lepb200_host_lep_generic(lepb200_lep* h, int zlib0, const uint8_t** data, size_t* len);
/* diagnostic: wall-clock seconds of the host front end alone over a batch with `threads` workers */
double lepb200_host_frontend_seconds(const lepb200_buffer* jpegs, int n, int threads, int32_t* first_error);

#ifdef __cplusplus
}
#endif
#endif /* LEPTON_B200_H_ */
