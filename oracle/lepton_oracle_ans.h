/* lepton_oracle_ans.h -- TEST INFRASTRUCTURE ONLY: the oracle's rANS coder (container version 3, the reference's -ans).
 *
 * Makefile.ans builds liblepton_oracle_ans.so from a copy of lepton_oracle.c in which this header is included right in front
 * of code_bit, and code_bit is renamed code_bit_bool (unused).  So the copy codes every decision through the code_bit below:
 * the grammar, the predictors and the model layout are lepton_oracle.c's, the coder and the branch update are these.
 * The state of the coder lives in g_ans (one segment at a time; lepton_oracle_ans.c sets it up). */

/* adv_record_obs_and_update (branch.hh:60-77), the update of the rANS coder's model (ans_bool_reader.hh:106,
 * ans_bool_writer.hh:62): from 255 the observed count restarts at 129 and only the other one is halved; the probability has
 * its low bit set.  Counts (1, 1) are never reached again, so only a branch never updated has the probability 128. */
static inline void branch_update_ans(Branch *b, int obs) {
    uint8_t *c = obs ? &b->c1 : &b->c0, *o = obs ? &b->c0 : &b->c1;
    if (*c == 0xff) { *c = 129; *o = (uint8_t)((1 + (unsigned)*o) >> 1); }
    else ++*c;
    b->p = (uint8_t)((((unsigned)b->c0 << 8) / ((unsigned)b->c0 + b->c1)) | 1);
}

/* ------------------------------------------------------------------ rANS coder (container version 3)
 * The reference's -ans streams (src/vp8/decoder/ans_bool_reader.hh:75-108, src/vp8/encoder/ans_bool_writer.hh:43-107,
 * src/ans/rans64.hh:60-139), restated from their description.  Two 64-bit states take turns decision by decision; a decision
 * at 8-bit probability p splits [0, 256) into [0, p) for bit 0 and [p, 256) for bit 1.  The stream is a sequence of
 * little-endian 32-bit words; the decoder reads them in order, zero past the end of the stream. */
#define ANS_L (1ull << 31)       /* lower bound of a normalised state (RANS64_L) */
typedef struct { uint64_t x0, x1; const uint8_t *p, *end; } AnsReader;

static uint32_t ar_word(AnsReader *r) {
    uint32_t w = 0;
    for (int k = 0; k < 4; ++k) if (r->p + k < r->end) w |= (uint32_t)r->p[k] << (8 * k);
    r->p += 4;
    return w;
}
static void ar_init(AnsReader *r, const uint8_t *p, size_t n) {
    r->p = p; r->end = p + n;
    r->x0 = ar_word(r); r->x0 |= (uint64_t)ar_word(r) << 32;    /* state of the first decision: words 0-1, low word first */
    r->x1 = ar_word(r); r->x1 |= (uint64_t)ar_word(r) << 32;    /* of the second: words 2-3 */
}
static int ar_read(AnsReader *r, int prob) {
    uint64_t x = r->x0;
    r->x0 = r->x1;
    const uint32_t cf = (uint32_t)(x & 255), p = (uint32_t)prob;
    const int bit = cf >= p;
    const uint32_t start = bit ? p : 0, freq = bit ? 256 - p : p;
    x = (uint64_t)freq * (x >> 8) + cf - start;
    if (x < ANS_L) x = (x << 32) | ar_word(r);                  /* at most one word per decision */
    r->x1 = x;
    return bit;
}

/* The writer codes the decisions in reverse.  Decisions 2k and 2k + 1 form pair k; the even one goes to state B (the state
 * the decoder starts with), the odd one to state A.  An odd count is completed by a pad decision (p = 1, bit 1), and four
 * pairs of (p = 128, bit 0) follow the last pair.  The pairs are coded last to first, A before B; a state at or above
 * ((L >> 8) << 32) * freq first emits its low word.  The emitted words are prepended, then A's and B's final states (low
 * word first, B in front), and the stream ends with the 4 bytes 00 80 00 80 (the reference's output includes one unused
 * pair of its symbol buffer: a (p = 128, bit 0) pair as two {bit, p} bytes each). */
static void aw_put(uint64_t *x, uint32_t *words, size_t *nw, uint32_t prob, int bit) {
    const uint32_t start = bit ? prob : 0, freq = bit ? 256 - prob : prob;
    uint64_t v = *x;
    if (v >= ((ANS_L >> 8) << 32) * freq) { words[(*nw)++] = (uint32_t)v; v >>= 32; }
    *x = ((v / freq) << 8) + (v % freq) + start;
}
/* tokens: prob | bit << 8.  Returns 0, LO_ASSERTION_FAILURE for a token of probability 0 (the reference's writer asserts),
 * or LO_OUTPUT_OVERFLOW when the stream does not fit `cap` (then *out_len = 0). */
int lo_ans_encode(const uint16_t *tokens, size_t n, uint8_t *out, size_t cap, size_t *out_len) {
    *out_len = 0;
    for (size_t i = 0; i < n; ++i) if ((tokens[i] & 0xff) == 0) return LO_ASSERTION_FAILURE;
    const size_t npairs = (n + 1) / 2 + 4;
    uint32_t *words = (uint32_t *)malloc((2 * npairs + 8) * sizeof(uint32_t));
    size_t nw = 0;
    uint64_t a = ANS_L, b = ANS_L;
    for (size_t k = npairs; k-- > 0;) {
        uint32_t pa = 128, pb = 128; int ba = 0, bb = 0;     /* the trailing (p = 128, bit 0) pairs */
        if (2 * k < n) {
            pb = tokens[2 * k] & 0xff; bb = (tokens[2 * k] >> 8) & 1;
            if (2 * k + 1 < n) { pa = tokens[2 * k + 1] & 0xff; ba = (tokens[2 * k + 1] >> 8) & 1; }
            else { pa = 1; ba = 1; }                          /* pad of an odd count */
        }
        aw_put(&a, words, &nw, pa, ba);
        aw_put(&b, words, &nw, pb, bb);
    }
    const size_t total = (4 + nw + 1) * 4;
    if (total > cap) { free(words); return LO_OUTPUT_OVERFLOW; }
    uint32_t head[4] = {(uint32_t)b, (uint32_t)(b >> 32), (uint32_t)a, (uint32_t)(a >> 32)};
    size_t o = 0;
    for (int i = 0; i < 4; ++i, o += 4) for (int k = 0; k < 4; ++k) out[o + k] = (uint8_t)(head[i] >> (8 * k));
    for (size_t i = nw; i-- > 0; o += 4) for (int k = 0; k < 4; ++k) out[o + k] = (uint8_t)(words[i] >> (8 * k));
    out[o] = 0x00; out[o + 1] = 0x80; out[o + 2] = 0x00; out[o + 3] = 0x80;
    *out_len = total;
    free(words);
    return 0;
}

/* One decision of a decode, as lo_decode_segment_ans_trace records it (test infrastructure: to build streams whose
 * decisions land on chosen states, and to show that a corpus reaches an edge of the coder). */
typedef struct {
    uint64_t x_before;                     /* the state the decision reads (its low byte against the probability) */
    uint64_t x_after;                      /* that state advanced, refilled when it fell below 2^31: the state two decisions on */
    int64_t word_off;                      /* byte offset in the stream of the word the refill took; -1: no refill */
    uint8_t prob, bit;                     /* the model's probability, the decoded bit */
    uint8_t c0, c1;                        /* the branch counts before the update (1..255) */
    uint8_t pad[4];
} lo_ans_step;

/* the coder of the segment in progress */
static struct {
    AnsReader ar;                          /* decode */
    const uint8_t *base;                   /* decode: start of the stream */
    lo_ans_step *trace; size_t ntrace, trace_cap;   /* decode, optional: the first trace_cap decisions */
    uint16_t *tok; size_t ntok, tok_cap;   /* encode: the decisions (prob | bit << 8), coded at the end in reverse */
} g_ans;

/* ANSBoolReader::get / ANSBoolWriter::put (ans_bool_reader.hh:87-108, ans_bool_writer.hh:43-64) */
static inline int code_bit(Codec *c, Branch *b, int bit) {
    if (c->encode) {
        if (g_ans.ntok == g_ans.tok_cap) {
            g_ans.tok_cap = g_ans.tok_cap ? 2 * g_ans.tok_cap : 4096;
            g_ans.tok = (uint16_t *)realloc(g_ans.tok, g_ans.tok_cap * sizeof(uint16_t));
        }
        g_ans.tok[g_ans.ntok++] = (uint16_t)(b->p | bit << 8);
    } else if (g_ans.ntrace < g_ans.trace_cap) {
        lo_ans_step *t = &g_ans.trace[g_ans.ntrace++];
        const uint8_t *p0 = g_ans.ar.p;
        t->x_before = g_ans.ar.x0;
        t->prob = b->p; t->c0 = b->c0; t->c1 = b->c1;
        bit = ar_read(&g_ans.ar, b->p);
        t->bit = (uint8_t)bit;
        t->x_after = g_ans.ar.x1;
        t->word_off = g_ans.ar.p != p0 ? (int64_t)(p0 - g_ans.base) : -1;
    } else {
        bit = ar_read(&g_ans.ar, b->p);
    }
    branch_update_ans(b, bit);
    c->ndecisions++;
    return bit;
}

