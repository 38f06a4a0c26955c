// emu_ans_encode.cc -- the encode side of container version 3 (rANS) on the CPU under the warp emulator of cuda_shim.h (test
// infrastructure): kernel A with the rANS model and the rANS pass (lep_encode.cu), launched the way
// lepb200_encode_launch_symbolise / lepb200_encode_launch_rangecode launch them (lep_capi.cu): one kernel A launch per
// coder, the bool-coded segments' range coder over segs[0 .. order_ans), the rANS pass over the rest.  Built on the harness
// of emu_kernels.cc (its launch helpers and range coder sequence), into a library of its own.
#include "emu_kernels.cc"

namespace {

struct AnsArgs {
    int stage;                       // 0 kernel A with the rANS model, 1 the rANS pass
    const ImageDesc* images; SegDesc* segs; int nseg; const int* order; int* counter;
    uint16_t* models; uint8_t* rows; size_t row_stride; uint16_t* tokens;
};

void ans_body(void* p) {
    const AnsArgs& a = *static_cast<const AnsArgs*>(p);
    if (a.stage == 0) lep_encode_kernel<EncAns>(a.images, a.segs, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride, a.tokens);
    else lep_anspass_kernel(a.segs, a.nseg, a.order, a.tokens);
}

void run_ans_pass(SegDesc* segs, int n, const int* order, uint16_t* tokens) {
    if (n <= 0) return;
    AnsArgs a;
    memset(&a, 0, sizeof(a));
    a.stage = 1; a.segs = segs; a.nseg = n; a.order = order; a.tokens = tokens;
    emu::launch((unsigned)((n + ANS_THREADS - 1) / ANS_THREADS), ANS_THREADS, ans_body, &a);
}

}  // namespace

// emu_encode_images with the coder of every image (coders[i], LEPB200_CODER_*; nullptr = all bool).  kernel: the bool
// part's range coder as in emu_encode_images (0 / 2 parallel, 1 serial).  Outputs in the caller's order (image after image),
// like lepb200_encode_fetch returns them; tok_caps (optional) receives every segment's token slot.
extern "C" int emu_encode_images_coded(int kernel, int grid_cap, int reverse, const lepb200_image* images, int nimages, const uint8_t* coders,
                                       lepb200_stream* out, uint8_t* arena, size_t arena_cap, uint32_t* tok_caps) {
    if (!out || !arena || (kernel != 0 && kernel != 1 && kernel != 2)) return LEPB200_ERR_INVALID;
    BatchPlan b;
    if (plan_batch(b, images, nimages, true, nullptr, coders)) return LEPB200_ERR_INVALID;
    const int nseg = (int)b.segs.size(), nbool = b.order_ans;
    emu::g_reverse = reverse != 0;
    std::vector<uint8_t> pv, sv;
    uint8_t* pbase = host_arena(pv, b.plane_total, 0);
    uint8_t* sbase = host_arena(sv, b.stream_total, 0);
    for (int i = 0; i < nimages; ++i)
        for (int c = 0; c < images[i].ncmp; ++c) memcpy(pbase + b.images[i].plane[c], images[i].planes[c], b.plane_bytes[(size_t)i * 3 + c]);
    rebase(b, pbase, sbase);
    std::vector<SegDesc>& segs = b.segs;

    EncArgs a;
    memset(&a, 0, sizeof(a));
    a.images = b.images.data(); a.segs = segs.data(); a.nseg = nseg; a.order = b.order.data(); a.row_stride = b.row_stride;
    int counter = 0;
    unsigned long long total_tokens = b.token_total;
    a.counter = &counter; a.total = &total_tokens;
    if (!b.tokens_known) {
        a.stage = 0; emu::launch((unsigned)nseg, CNT_THREADS, enc_body, &a);
        a.stage = 1; emu::launch(1, 1024, enc_body, &a);
    }
    std::vector<uint16_t> tokens((size_t)total_tokens + 128, 0);
    a.tokens = tokens.data();
    std::vector<uint16_t> models;
    std::vector<uint8_t> rows;
    for (int part = 0; part < 2; ++part) {
        const int first = part == 0 ? 0 : nbool, n = part == 0 ? nbool : nseg - nbool;
        if (n == 0) continue;
        unsigned grid = (unsigned)((n + ENC_WARPS_PER_CTA - 1) / ENC_WARPS_PER_CTA);
        if (grid_cap > 0) grid = std::min(grid, (unsigned)grid_cap);
        models.assign((size_t)grid * ENC_WARPS_PER_CTA * M_TOTAL, 0x5a5a);      // the kernel clears its own
        rows.assign((size_t)grid * ENC_WARPS_PER_CTA * b.row_stride, 0);
        counter = 0;
        if (part == 0) {
            a.models = models.data(); a.rows = rows.data(); a.nseg = n; a.order = b.order.data();
            a.stage = 2; emu::launch(grid, ENC_WARPS_PER_CTA * 32, enc_body, &a);
        } else {
            AnsArgs x;
            x.stage = 0; x.images = b.images.data(); x.segs = segs.data(); x.nseg = n; x.order = b.order.data() + first; x.counter = &counter;
            x.models = models.data(); x.rows = rows.data(); x.row_stride = b.row_stride; x.tokens = tokens.data();
            emu::launch(grid, ENC_WARPS_PER_CTA * 32, ans_body, &x);
        }
    }
    std::vector<uint8_t> ovf;
    if (nbool > 0) {
        a.nseg = nbool; a.order = b.order.data();
        run_range_coder(kernel, a, total_tokens, ovf);
    }
    run_ans_pass(segs.data(), nseg - nbool, b.order.data() + nbool, tokens.data());
    emu::g_reverse = false;
    size_t used = 0;
    for (int d = 0; d < nseg; ++d) {
        const int s = b.seg_out.empty() ? d : b.seg_out[d];
        const size_t n = segs[d].status == 0 ? segs[d].len : 0;
        if (used + n > arena_cap) return LEPB200_ERR_NOMEM;
        memcpy(arena + used, reinterpret_cast<const uint8_t*>(segs[d].stream), n);
        if (tok_caps) tok_caps[s] = segs[d].tok_cap;
        out[s].data = arena + used;
        out[s].len = n;
        out[s].status = segs[d].status;
        out[s].reserved = 0;
        out[s].ndecisions = (uint64_t)segs[d].ndecisions_lo | ((uint64_t)segs[d].ndecisions_hi << 32);
        used += n;
    }
    return 0;
}

// The rANS pass alone on caller token streams: segment s has ntok[s] tokens (prob | bit << 8, back to back in `tokens`)
// and a token slot of tok_cap[s] tokens (0: token_slot(ntok[s]), as the library gives it), laid out one after the other with
// 64 canary tokens (0xC3C3) in front of the first slot and behind every slot; segments run longest first.  Outputs per
// segment: status, len, the bytes back to back in `out`; *canary_bad = canary tokens that changed.
extern "C" int emu_ans_pass(int reverse, int nseg, const uint16_t* tokens, const uint32_t* ntok, const uint32_t* tok_cap,
                            int32_t* status_out, uint32_t* len_out, uint8_t* out, size_t out_cap, uint64_t* canary_bad) {
    if (nseg <= 0 || !tokens || !ntok || !out || !canary_bad) return LEPB200_ERR_INVALID;
    constexpr uint32_t CANARY = 64;
    constexpr uint16_t CANARY_TOKEN = 0xC3C3;
    std::vector<SegDesc> segs(nseg);
    unsigned long long total = CANARY;
    for (int s = 0; s < nseg; ++s) {
        SegDesc& sd = segs[s];
        memset(&sd, 0, sizeof(sd));
        sd.ntok = ntok[s];
        sd.tok_cap = tok_cap && tok_cap[s] ? tok_cap[s] : token_slot(ntok[s]);
        sd.tokens = total;
        total += (sd.tok_cap + CANARY + 63) / 64 * 64;               // slots start 128-byte aligned, as lep_token_offsets_kernel lays them out
    }
    std::vector<uint16_t> tok((size_t)total + 128, CANARY_TOKEN);
    uint16_t* base = reinterpret_cast<uint16_t*>(align_up((size_t)(uintptr_t)tok.data(), 128));
    size_t src = 0;
    for (int s = 0; s < nseg; ++s) {
        uint16_t* slot = base + segs[s].tokens;
        for (uint32_t k = 0; k < segs[s].tok_cap; ++k) slot[k] = 0;
        if (segs[s].ntok) memcpy(slot, tokens + src, (size_t)segs[s].ntok * 2);
        src += ntok[s];
    }
    std::vector<int> order(nseg);
    for (int i = 0; i < nseg; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return ntok[x] > ntok[y]; });
    emu::g_reverse = reverse != 0;
    run_ans_pass(segs.data(), nseg, order.data(), base);
    emu::g_reverse = false;
    uint64_t bad = 0;
    for (uint32_t k = 0; k < CANARY; ++k) bad += base[k] != CANARY_TOKEN;
    for (int s = 0; s < nseg; ++s) {
        const uint16_t* slot = base + segs[s].tokens;
        const uint32_t end = (uint32_t)((segs[s].tok_cap + CANARY + 63) / 64 * 64);
        for (uint32_t k = segs[s].tok_cap; k < end; ++k) bad += slot[k] != CANARY_TOKEN;
    }
    size_t used = 0;
    for (int s = 0; s < nseg; ++s) {
        const size_t n = segs[s].status == 0 ? segs[s].len : 0;
        if (used + n > out_cap) return LEPB200_ERR_NOMEM;
        memcpy(out + used, reinterpret_cast<const uint8_t*>(segs[s].stream), n);
        used += n;
        status_out[s] = segs[s].status;
        len_out[s] = (uint32_t)n;
    }
    *canary_bad = bad;
    return 0;
}

// The rANS pass's division (ans_divide with the table entries ans_recip / ans_recip_shift): q[i] = x[i] / f[i],
// r[i] = x[i] % f[i] for x[i] < 2^63, f[i] in [1, 256].
extern "C" void emu_ans_divide(int n, const unsigned long long* x, const uint32_t* f, unsigned long long* q, uint32_t* r) {
    for (int i = 0; i < n; ++i) q[i] = ans_divide(x[i], f[i], ans_recip(f[i]), ans_recip_shift(f[i]), r[i]);
}

// ans_stream_bound / ans_slot_fits of the library (lep_encode.cu)
extern "C" unsigned long long emu_ans_stream_bound(unsigned long long ntok) { return ans_stream_bound(ntok); }
extern "C" int emu_ans_slot_fits(unsigned long long ntok, unsigned long long tok_cap) { return ans_slot_fits(ntok, tok_cap) ? 1 : 0; }

// One decision of the rANS pass (ans_put) on state x[i] with token tok[i]: the state after it, and the word it emitted
// (emitted[i] = 1) or none.
extern "C" void emu_ans_put(int n, const unsigned long long* x, const uint16_t* tok, unsigned long long* x_out, uint32_t* word, uint8_t* emitted) {
    unsigned long long s_m[256];
    for (uint32_t f = 1; f <= 256; ++f) s_m[f - 1] = ans_recip(f);
    for (int i = 0; i < n; ++i) {
        uint32_t bad = 0, buf[2] = {0, 0};
        uint32_t* wp = buf + 1;
        unsigned long long v = x[i];
        ans_put(v, ans_token(tok[i], s_m, bad), wp);
        x_out[i] = v;
        emitted[i] = wp != buf + 1;
        word[i] = buf[0];
    }
}
