// emu_zlib0.cc -- the emulator build of the zlib0 tests: emu_kernels.cc plus an entry point that runs lep_huffencode_kernel
// like emu_huffman_encode does and also hands back where each thread-segment wrote and the Adler-32 it took over those bytes.
// reverse = 1 runs the launch's CTAs and threads in reverse order (emu::g_reverse).
#include "emu_kernels.cc"

extern "C" int emu_huffman_encode_adler(const lepb200_henc_image* im, int ncmp, int mcuv, const int16_t* const* planes, const int* bch,
                                        int reverse, uint8_t* out, int32_t* seg_status, uint32_t* seg_off, uint32_t* seg_produced,
                                        uint32_t* seg_adler) {
    if (!im || !planes || !bch || !out || im->scan_bytes == 0 || im->nseg < 1 || im->nseg > LEPB200_MAX_SEGMENTS) return LEPB200_ERR_INVALID;
    HEncImage d;
    memset(&d, 0, sizeof(d));
    std::vector<HEncTable> tabs;
    d.ncmp = ncmp; d.mcuv = mcuv; d.rsti = im->rsti; d.padbit = im->padbit; d.scan_len = im->scan_bytes;
    for (int c = 0; c < ncmp; ++c) {
        d.H[c] = im->H[c]; d.V[c] = im->V[c]; d.bch[c] = bch[c];
        d.plane[c] = (unsigned long long)(uintptr_t)planes[c];
        HEncTable t;
        if (!emu_build_enc_table(im->dc[c], t)) return LEPB200_ERR_INVALID;
        d.dc_tab[c] = (int)tabs.size(); tabs.push_back(t);
        if (!emu_build_enc_table(im->ac[c], t)) return LEPB200_ERR_INVALID;
        d.ac_tab[c] = (int)tabs.size(); tabs.push_back(t);
    }
    d.mcuh = bch[0] / im->H[0];
    std::vector<uint8_t> obuf((size_t)im->scan_bytes + 256 + 512, 0xA5);
    uint8_t* obase = reinterpret_cast<uint8_t*>(align_up((size_t)(uintptr_t)obuf.data(), 256));
    d.out = (unsigned long long)(uintptr_t)obase;
    std::vector<HEncSeg> segs;
    uint32_t off = 0;
    for (int k = 0; k < im->nseg; ++k) {
        HEncSeg sg;
        memset(&sg, 0, sizeof(sg));
        sg.image = 0; sg.my0 = im->seg[k].mcu_row_start; sg.my1 = im->seg[k].mcu_row_end;
        for (int c = 0; c < 3; ++c) sg.lastdc[c] = im->seg[k].last_dc[c];
        sg.ov_bits = im->seg[k].overhang_bits; sg.ov_byte = im->seg[k].overhang_byte;
        sg.out_off = off; sg.expect = im->seg[k].expect_bytes; sg.is_last = k + 1 == im->nseg;
        off += im->seg[k].expect_bytes;
        segs.push_back(sg);
    }
    HEncArgs a{&d, segs.data(), (int)segs.size(), tabs.data()};
    emu::g_reverse = reverse != 0;
    emu::launch((unsigned)((segs.size() + HENC_WARPS - 1) / HENC_WARPS), HENC_WARPS * 32, henc_body, &a);
    emu::g_reverse = false;
    memcpy(out, obase, im->scan_bytes);
    for (int k = 0; k < im->nseg; ++k) {
        seg_status[k] = segs[k].status; seg_off[k] = segs[k].out_off; seg_produced[k] = segs[k].produced; seg_adler[k] = segs[k].adler;
    }
    return 0;
}
