/* lepton_oracle_ans.c -- TEST INFRASTRUCTURE ONLY: lepton_oracle.c with the rANS coder of container version 3 (the
 * reference's -ans: src/vp8/decoder/ans_bool_reader.hh, src/vp8/encoder/ans_bool_writer.hh, src/ans/rans64.hh) in place of
 * the bool coder.  The copy of lepton_oracle.c that Makefile.ans generates codes every decision through lepton_oracle_ans.h.
 * Exports lo_encode_segment_ans / lo_decode_segment_ans (no marker bit, no stop bits), lo_decode_segment_ans_trace (the
 * decode with a record of every decision) and lo_ans_encode (the writer alone). */
#include "lepton_oracle_ans_gen.c"

int lo_encode_segment_ans(const lo_geometry *g, const int16_t *const planes[3], int min_y, int max_y, int is_last,
                          uint8_t *out, size_t cap, size_t *out_len, uint64_t *ndecisions) {
    Codec c;
    *out_len = 0;
    g_ans.ntok = 0;
    int e = codec_init(&c, g, (int16_t *const *)planes, 1);
    if (e) { codec_free(&c); return e; }
    e = code_segment(&c, min_y, max_y, is_last);
    if (!e) e = lo_ans_encode(g_ans.tok, g_ans.ntok, out, cap, out_len);
    if (ndecisions) *ndecisions = c.ndecisions;
    codec_free(&c);
    return e;
}

/* lo_decode_segment_ans that also records its first trace_cap decisions in trace (lo_ans_step, lepton_oracle_ans.h). */
int lo_decode_segment_ans_trace(const lo_geometry *g, int16_t *const planes[3], int min_y, int max_y, int is_last,
                                const uint8_t *in, size_t in_len, uint64_t *ndecisions, lo_ans_step *trace, size_t trace_cap) {
    Codec c;
    int e = codec_init(&c, g, planes, 0);
    if (e) { codec_free(&c); return e; }
    ar_init(&g_ans.ar, in, in_len);
    g_ans.base = in;
    g_ans.trace = trace; g_ans.ntrace = 0; g_ans.trace_cap = trace ? trace_cap : 0;
    e = code_segment(&c, min_y, max_y, is_last);
    g_ans.trace = NULL; g_ans.trace_cap = 0;
    if (ndecisions) *ndecisions = c.ndecisions;
    codec_free(&c);
    return e;
}

int lo_decode_segment_ans(const lo_geometry *g, int16_t *const planes[3], int min_y, int max_y, int is_last,
                          const uint8_t *in, size_t in_len, uint64_t *ndecisions) {
    return lo_decode_segment_ans_trace(g, planes, min_y, max_y, is_last, in, in_len, ndecisions, NULL, 0);
}
