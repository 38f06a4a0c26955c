// b200_component_coders.hh -- the reference-side binding of lepton-b200: BaseEncoder / BaseDecoder adapters that a
// maintainer of dropbox/lepton compiles INTO the reference (next to src/lepton/simple_encoder.hh, the existing proof
// that the boundary is pluggable) and links with -llepton_b200.  Nothing else of the reference changes except the two
// factory lines quoted at the bottom.
//
//   B200ComponentEncoder::encode_chunk  replaces VP8ComponentEncoder::vp8_full_encoder
//                                       (src/lepton/vp8_encoder.cc:521-614; interface src/lepton/base_coders.hh:59-62)
//   B200ComponentDecoder::decode_chunk  replaces VP8ComponentDecoder::decode_chunk (src/lepton/vp8_decoder.cc:387-490)
//                                       on the full-plane path the reference takes for progressive files and with
//                                       -forceprogressive (jpgcoder.cc:1052-1055, :4359-4360)
//   B200ComponentDecoder::initialize_baseline_decoder + decode_row  replace the row-by-row baseline entry
//                                       (vp8_decoder.cc:314-371, lepton_codec.cc:7-47; caller recoder.cc:472-545, :728)
//
// This file includes the reference's headers, so it is compiled only where they exist: tests/test_adapter_compiles.py
// checks it against /root/reference with the reference's own flags (-std=c++11 -fno-exceptions -fno-rtti).
#ifndef LEPB200_COMPONENT_CODERS_HH_
#define LEPB200_COMPONENT_CODERS_HH_

#include <algorithm>
#include <cstring>
#include <vector>

#include "base_coders.hh"                 // src/lepton
#ifndef LEPB200_HAVE_UNCOMPRESSED_COMPONENTS  // (that header has no include guard: a file that already included it says so)
#include "uncompressed_components.hh"     // src/lepton
#endif
#include "../io/MuxReader.hh"
#include "../io/ioutil.hh"
#include "../vp8/util/memory.hh"

#include "lepton_b200.h"

extern unsigned char ujgversion;          // src/lepton/jpgcoder.cc:544

namespace lepb200_adapter {

// UncompressedComponents -> lepb200_image (the same fields, plain C).  `planes` are the reference's own buffers:
// BlockBasedImage is a row-major array of AlignedBlock (src/vp8/util/block_based_image.hh:52-75).
template <class Components>
inline void fill_image(lepb200_image& im, Components* c, bool writable) {
    memset(&im, 0, sizeof(im));
    im.ncmp = c->get_num_components();
    im.mcuv = c->get_mcu_count_vertical();
    Sirikata::Array1d<uint32_t, (size_t)ColorChannel::NumBlockTypes> maxh = c->get_max_coded_heights();
    for (int k = 0; k < im.ncmp; ++k) {
        const BlockBasedImage& p = c->full_component_nosync(k);
        im.bch[k] = (int32_t)p.block_width();
        im.bcv[k] = (int32_t)p.original_height();
        im.trunc_bcv[k] = (int32_t)maxh[k];
        im.trunc_bc[k] = (int32_t)c->component_size_in_blocks(k);
        memcpy(im.qtable_zigzag[k], c->get_quantization_tables((BlockType)k), 64 * sizeof(uint16_t));
        im.planes[k] = const_cast<int16_t*>(p.raster(0).raw_data());
    }
    (void)writable;
}

inline void exit_on(int api_rc) {
    if (api_rc == LEPB200_ERR_NOMEM) custom_exit(ExitCode::OOM);
    if (api_rc != LEPB200_OK) custom_exit(ExitCode::OS_ERROR);
}

}  // namespace lepb200_adapter

class B200ComponentEncoder : public BaseEncoder {
    lepb200_ctx* ctx_;
public:
    B200ComponentEncoder() : ctx_(NULL) { lepb200_adapter::exit_on(lepb200_create(&ctx_, 0)); }
    ~B200ComponentEncoder() { lepb200_destroy(ctx_); }
    void registerWorkers(GenericWorker*, unsigned int) {}         // CUDA replaces the spin workers
    size_t get_decode_model_memory_usage() const { return 0; }    // the models live in HBM, not in the jailed heap
    size_t get_decode_model_worker_memory_usage() const { return 0; }

    CodingReturnValue encode_chunk(const UncompressedComponents* input, IOUtil::FileWriter* out,
                                   const ThreadHandoff* selected_splits, unsigned int num_selected_splits) {
        if (num_selected_splits == 0 || num_selected_splits > LEPB200_MAX_SEGMENTS) custom_exit(ExitCode::ASSERTION_FAILURE);
        lepb200_image im;
        lepb200_adapter::fill_image(im, input, false);
        im.nseg = (int32_t)num_selected_splits;
        for (unsigned i = 0; i < num_selected_splits; ++i) im.luma_y_start[i] = selected_splits[i].luma_y_start;
        lepb200_stream s[LEPB200_MAX_SEGMENTS];
#ifdef ENABLE_ANS_EXPERIMENTAL
        // -ans (container version 3, jpgcoder.cc:1704-1705): rANS-coded segment streams
        const uint8_t coder = ujgversion == 3 ? LEPB200_CODER_ANS : LEPB200_CODER_BOOL;
        lepb200_adapter::exit_on(lepb200_encode_images_coded(ctx_, &im, 1, &coder, s));
#else
        lepb200_adapter::exit_on(lepb200_encode_images(ctx_, &im, 1, s));
#endif
        for (unsigned i = 0; i < num_selected_splits; ++i) {
            if (s[i].status) custom_exit((ExitCode)s[i].status);   // the reference's own ExitCode values
        }
        // the tail of vp8_full_encoder, unchanged in meaning (vp8_encoder.cc:573-614): interleave the segment
        // streams through the reference's MuxWriter (256 B, then 4096 B, then 64 KiB per turn), close, LE32 size
        Sirikata::MuxWriter mux(out, Sirikata::JpegAllocator<uint8_t>(), ujgversion);
        size_t off[LEPB200_MAX_SEGMENTS] = {0};
        bool any = true;
        while (any) {
            any = false;
            for (unsigned i = 0; i < num_selected_splits; ++i) {
                if (s[i].len <= off[i]) continue;
                any = true;
                const size_t turn = off[i] == 0 ? 256 : (off[i] == 256 ? 4096 : 65536);
                const size_t n = std::min<size_t>(turn, (size_t)s[i].len - off[i]);
                off[i] += mux.Write((uint8_t)i, s[i].data + off[i], (unsigned int)n).first;
            }
        }
        mux.Close();
        uint32_t size = (uint32_t)out->getsize() + 4;
        const uint8_t le[4] = {(uint8_t)size, (uint8_t)(size >> 8), (uint8_t)(size >> 16), (uint8_t)(size >> 24)};
        out->Write(le, 4);
        return CODING_DONE;
    }
};

class B200ComponentDecoder : public BaseDecoder {
    lepb200_ctx* ctx_;
    Sirikata::DecoderReader* in_;
    std::vector<ThreadHandoff> handoffs_;
    std::vector<int16_t> rows_[4];          // baseline entry: the decoded planes rows are served from
    uint32_t rows_bch_[4];
    std::vector<NeighborSummary> dummy_;     // off_y() wants a neighbour-summary iterator; only the block pointer is used
    GenericWorker* workers_;
    unsigned int num_workers_;

    // All thread-segments of the image in one launch: demux with the reference's own MuxReader
    // (src/io/MuxReader.hh:230-331; it stops at the EOF marker or, for version 1, when the bounded reader runs dry,
    // jpgcoder.cc:2176), then lepb200_decode_images into im.planes.
    void decode_all(lepb200_image& im) {
        const int nseg = (int)handoffs_.size();
        if (nseg == 0 || nseg > LEPB200_MAX_SEGMENTS) custom_exit(ExitCode::VERSION_UNSUPPORTED);   // legacy files: no handoff table
        Sirikata::MuxReader mux(Sirikata::JpegAllocator<uint8_t>(), nseg, 0, in_);
        std::pair<Sirikata::MuxReader::ResizableByteBuffer::const_iterator,
                  Sirikata::MuxReader::ResizableByteBuffer::const_iterator> seg[Sirikata::MuxReader::MAX_STREAM_ID];
        mux.fillBufferEntirely(seg);
        im.nseg = nseg;
        lepb200_stream s[LEPB200_MAX_SEGMENTS];
        memset(s, 0, sizeof(s));
        for (int i = 0; i < nseg; ++i) {
            im.luma_y_start[i] = handoffs_[i].luma_y_start;
            s[i].data = seg[i].first;
            s[i].len = (uint64_t)(seg[i].second - seg[i].first);
        }
        int32_t st[LEPB200_MAX_SEGMENTS];
#ifdef ENABLE_ANS_EXPERIMENTAL
        // a version-3 file's streams are rANS-coded (the reference's makeDecoder(..., ujgversion == 3), jpgcoder.cc:1727);
        // every decoder entry (decode_chunk, the row entry, -singlethread) comes through here
        const uint8_t coder = ujgversion == 3 ? LEPB200_CODER_ANS : LEPB200_CODER_BOOL;
        lepb200_adapter::exit_on(lepb200_decode_upload_coded(ctx_, &im, 1, s, &coder));
        lepb200_adapter::exit_on(lepb200_decode_launch(ctx_));
        lepb200_adapter::exit_on(lepb200_decode_fetch(ctx_, &im, 1, st));
#else
        lepb200_adapter::exit_on(lepb200_decode_images(ctx_, &im, 1, s, st));
#endif
        for (int i = 0; i < nseg; ++i) {
            if (st[i]) custom_exit((ExitCode)st[i]);
        }
    }
public:
    B200ComponentDecoder() : ctx_(NULL), in_(NULL), workers_(NULL), num_workers_(0) { lepb200_adapter::exit_on(lepb200_create(&ctx_, 0)); }
    ~B200ComponentDecoder() { lepb200_destroy(ctx_); }
    void initialize(Sirikata::DecoderReader* input, const std::vector<ThreadHandoff>& thread_transition_info) {
        in_ = input;
        handoffs_ = thread_transition_info;
    }
    // Full-plane entry (progressive files, -forceprogressive): planes go straight into the reference's own buffers.
    CodingReturnValue decode_chunk(UncompressedComponents* dst) {
        lepb200_image im;
        lepb200_adapter::fill_image(im, dst, true);
        decode_all(im);
        for (int k = 0; k < im.ncmp; ++k) dst->worker_mark_cmp_finished((BlockType)k);
        return CODING_DONE;
    }
    // Baseline entry (recode_baseline_jpeg, recoder.cc:694-889): the reference keeps only a 2-row framebuffer per
    // worker and pulls rows with decode_row from up to 8 threads while it Huffman-encodes.  Here the whole image is
    // decoded on the GPU when the decoder is set up -- a row-at-a-time launch would leave the device idle -- and
    // decode_row copies the requested row into the caller's ring (read-only on shared planes: safe from any thread).
    std::vector<ThreadHandoff> initialize_baseline_decoder(const UncompressedComponents* const colldata,
            Sirikata::Array1d<BlockBasedImagePerChannel<true>, MAX_NUM_THREADS>&) {
        lepb200_image im;
        memset(&im, 0, sizeof(im));
        im.ncmp = colldata->get_num_components();
        im.mcuv = colldata->get_mcu_count_vertical();
        Sirikata::Array1d<uint32_t, (size_t)ColorChannel::NumBlockTypes> maxh = colldata->get_max_coded_heights();
        uint32_t widest = 0;
        for (int k = 0; k < im.ncmp; ++k) {
            im.bch[k] = colldata->block_width(k);
            im.bcv[k] = colldata->block_height(k);
            im.trunc_bcv[k] = (int32_t)maxh[k];
            im.trunc_bc[k] = (int32_t)colldata->component_size_in_blocks(k);
            memcpy(im.qtable_zigzag[k], colldata->get_quantization_tables((BlockType)k), 64 * sizeof(uint16_t));
            rows_[k].assign((size_t)im.bch[k] * im.bcv[k] * 64, 0);
            rows_bch_[k] = (uint32_t)im.bch[k];
            im.planes[k] = rows_[k].data();
            widest = std::max(widest, rows_bch_[k]);
        }
        dummy_.resize((size_t)widest * 2 + 2);
        if (handoffs_.empty()) {
            // legacy container: segment count and luma split rows open the payload (vp8_decoder.cc:337-366); such
            // handoffs carry no Huffman state, so the caller re-encodes single-threaded (recoder.cc:731-733)
            unsigned char mark = 0;
            if (in_->Read(&mark, 1).second != Sirikata::JpegError::nil()) return handoffs_;
            if (mark == 0) custom_exit(ExitCode::THREADING_PARTIAL_MCU);
            ThreadHandoff th;
            memset(&th, 0, sizeof(th));
            th.num_overhang_bits = ThreadHandoff::LEGACY_OVERHANG_BITS;
            th.luma_y_end = colldata->block_height(0);
            handoffs_.insert(handoffs_.end(), mark, th);
            std::vector<uint16_t> ends(mark - 1);
            IOUtil::ReadFull(in_, ends.data(), sizeof(uint16_t) * (mark - 1));
            const int mul = colldata->min_vertical_luma_multiple();
            for (int i = 0; i + 1 < mark; ++i) {
                handoffs_[i].luma_y_end = htole16(ends[i]);
                if (handoffs_[i].luma_y_end % mul) custom_exit(ExitCode::THREADING_PARTIAL_MCU);
            }
            for (int i = 1; i < mark; ++i) handoffs_[i].luma_y_start = handoffs_[i - 1].luma_y_end;
        }
        decode_all(im);
        if (!handoffs_.empty()) handoffs_.back().luma_y_end = colldata->block_height(0);          // vp8_decoder.cc:367-369
        for (size_t i = 0; i + 1 < handoffs_.size(); ++i) {
            if (handoffs_[i].luma_y_end == 0) handoffs_[i].luma_y_end = handoffs_[i + 1].luma_y_start;
        }
        return handoffs_;
    }
    void decode_row(int, BlockBasedImagePerChannel<true>& image_data,
                    Sirikata::Array1d<uint32_t, (uint32_t)ColorChannel::NumBlockTypes> component_size_in_blocks,
                    int component, int curr_y) {
        const uint32_t w = rows_bch_[component];
        const size_t first = (size_t)curr_y * w;
        if (first >= (size_t)component_size_in_blocks[component]) return;                  // truncated image (lepton_codec.cc:21-24)
        const size_t n = std::min<size_t>(w, (size_t)component_size_in_blocks[component] - first);
        AlignedBlock* dst = image_data[component]->off_y(curr_y, dummy_.begin()).cur;          // row slot of the 2-row ring
        memcpy(dst->raw_data(), rows_[component].data() + first * 64, n * 64 * sizeof(int16_t));
    }
    // The spin workers belong to the caller's Huffman re-encoder (recoder.cc:765-815 hands them the per-thread recode
    // jobs through getWorker); the decoder only keeps them, as LeptonCodec does (lepton_codec.hh:182-185).
    void registerWorkers(GenericWorker* workers, unsigned int num_workers) { workers_ = workers; num_workers_ = num_workers; }
    GenericWorker* getWorker(unsigned int i) { return workers_ ? &workers_[i] : NULL; }
    unsigned int getNumWorkers() const { return num_workers_; }
    size_t get_model_memory_usage() const { return 0; }
    size_t get_model_worker_memory_usage() const { return 0; }
    void flush() {}
    void map_logical_thread_to_physical_thread(int, int) {}
    void clear_thread_state(int, int, BlockBasedImagePerChannel<true>&) {}
    void reset_all_comm_buffers() {}
};

// The lines that change in the reference (src/lepton/jpgcoder.cc; with -DENABLE_ANS_EXPERIMENTAL also :1705, the rANS
// encoder's  g_encoder.reset(makeEncoder<ANSBoolReader>(g_threaded, g_threaded));  ->  g_encoder.reset(new B200ComponentEncoder);):
//   :1710   g_encoder.reset(makeEncoder<VPXBoolReader>(g_threaded, g_threaded));   ->  g_encoder.reset(new B200ComponentEncoder);
//   :1727   g_decoder = makeDecoder(g_threaded, g_threaded, ujgversion == 3);       ->  g_decoder = new B200ComponentDecoder;
//           followed, as in makeBoth (:440-452), by  if (g_threaded) g_decoder->registerWorkers(get_worker_threads(NUM_THREADS), NUM_THREADS);
// and the process that owns the CUDA context runs with -unjailed (seccomp filter, src/io/Seccomp.cc:94-97).
#endif
