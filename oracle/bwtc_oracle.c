/*
 * oracle/bwtc_oracle.c -- CPU restatement of compressjs' BWTC container (SURVEY.md section 8 rows a20-a22).
 *
 * THIS IS TEST INFRASTRUCTURE, NOT THE PRODUCT (same rules as bz2_oracle.c).  There is no CUDA BWTC path yet:
 * the range coder and the adaptive model form one serial chain over the whole file.  The restatement exists so
 * that the block stages which DO run on the GPU (sentinel BWT, MTF, zero-run digits) have a container-level
 * checker, and as the CPU yardstick for BASELINE config 4.
 *
 * Restates, citing file:line under /root/reference:
 *   lib/BWTC.js:12-139   compressFile (levels 6..9: FenwickModel; levels 1..5: DefSumModel)
 *   lib/BWTC.js:141-231  decompressFile
 *   lib/RangeCoder.js:27-232
 *   lib/FenwickModel.js:15-165
 *   lib/DefSumModel.js:11-131
 *   lib/LogDistanceModel.js:8-49 over lib/NoModel.js:8-30 (raw bits through the range coder)
 *   lib/Util.js:105-220  magic + self-delimiting size + suppressed final byte
 *
 * Pinned against the vectors SURVEY.md section 8(c) lists for BWTC -9 (sample0 whole file in hex, sizes and
 * SHA-256 of sample1..5, README.md:41 size of sample5) -- tests/test_oracle.py.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_EXPORT __attribute__((visibility("default")))

int32_t orc_bwt_sentinel(const uint8_t* T, uint8_t* U, int32_t n);
int orc_unbwt_sentinel(const uint8_t* T, uint8_t* U, int32_t n, int32_t pidx);

/* ---- byte sink / source --------------------------------------------------------------------- */
typedef struct { uint8_t* p; size_t n, cap; int oom; } sink_t;
static void put(sink_t* s, uint32_t b) {
  if (s->n == s->cap) {
    size_t nc = s->cap ? s->cap * 2 : 4096;
    uint8_t* np = (uint8_t*)realloc(s->p, nc);
    if (!np) { s->oom = 1; return; }
    s->p = np; s->cap = nc;
  }
  s->p[s->n++] = (uint8_t)b;
}
typedef struct { const uint8_t* p; size_t n, pos; } src_t;
static int get(src_t* s) { return s->pos < s->n ? s->p[s->pos++] : -1; }  /* Stream.EOF = -1 */

static int fls32(uint32_t v) { int r = 0; while (v) { r++; v >>= 1; } return r; }  /* Util.js:301-316 */

/* ---- trace (orc_bwtc_compress_trace): counters beside the reference arithmetic, which they never change ---------- */
typedef struct {
  uint32_t n, alpha, nsym, ntriples;      /* raw bytes, used bytes, model symbols, coded triples (header included) */
  uint32_t rescales, rescales_esc;        /* Fenwick rescales; those triggered by the escape step of an escape */
  uint32_t rescales_ff00, rescales_noesc; /* ... at a total of exactly 0xFF00; ... with noEscape (the escape zeroed) */
  uint32_t escapes, last_escape;          /* symbols coded through the escape; the last escape (FenwickModel.js:68) */
  uint32_t reescapes, esc_lane31;         /* escapes of a symbol seen before in the block; escapes at symbol k = 31 mod 32 */
  uint32_t ds_rebuilds, ds_esc_cap;       /* deferred-sum table rebuilds; escapes not counted as update[esc] is 40 */
  uint32_t max_tot, carries;              /* largest tot_f; carries into the buffered byte */
  uint32_t help_carry, help_nocarry;      /* pending 0xFF bytes resolved with a carry (as 0x00) / without (as 0xFF) */
  uint32_t corr[3];                       /* steps of r = umulhi(range, 0xFFFFFFFF / tot) up to range / tot: 0, 1, 2 */
  uint32_t max_help;                      /* most bytes pending in the block */
  uint32_t help_in, resolved_in;          /* bytes pending when the block starts; how they came out: 1 as 0xFF, 2 as 0x00 */
  uint64_t help, bytes_out, bytecount;    /* the coder after the block's last triple: pending, stream bytes, bytecount */
} orc_bwtc_block_t;
typedef struct {
  uint32_t nblocks, max_help;
  uint32_t first_carry;                   /* the coder's first byte out (the size field's last group) carried */
  uint32_t finish_carry, finish_round;    /* finish: tmp > 0xFF; the rounding rule added one */
  uint32_t corr2;                         /* two correction steps anywhere in the file */
  uint64_t coder_bytes, bytecount;        /* bytes the coder put out; bytecount in the trailer */
} orc_bwtc_file_t;
static _Thread_local orc_bwtc_block_t* TRB;   /* the block being coded, or a scratch record outside blocks */
static _Thread_local orc_bwtc_file_t* TRF;
static _Thread_local uint8_t TR_SEEN[260];
#define TRC(x) do { if (TRB) { x; } } while (0)
static void tr_put(int carry) {
  if (!TRF) return;
  if (TRF->coder_bytes++ == 0) TRF->first_carry = (uint32_t)carry;
}
static void tr_tot(uint32_t range, uint32_t tot) {
  TRB->ntriples++;
  if (tot > TRB->max_tot) TRB->max_tot = tot;
  const uint32_t r0 = (uint32_t)(((uint64_t)range * (0xFFFFFFFFu / tot)) >> 32);
  const uint32_t k = range / tot - r0;
  TRB->corr[k < 2 ? k : 2]++;
  if (k >= 2) TRF->corr2++;
}

/* ---- range coder (RangeCoder.js) ---------------------------------------------------------------- */
#define TOP_VALUE 0x80000000u      /* 2^(CODE_BITS-1), :15 */
#define SHIFT_BITS 23              /* :16 */
#define EXTRA_BITS 7               /* (32-2)%8+1, :17 */
#define BOTTOM_VALUE (TOP_VALUE >> 8)

typedef struct {
  uint32_t low, range, buffer;
  uint64_t help;
  uint32_t bytecount;
  sink_t* out;
  src_t* in;
} rc_t;

static void enc_start(rc_t* rc, sink_t* out, uint32_t c, uint32_t initlength) {  /* :66-72 */
  rc->low = 0; rc->range = TOP_VALUE; rc->buffer = c; rc->help = 0; rc->bytecount = initlength; rc->out = out; rc->in = NULL;
}
static void enc_normalize(rc_t* rc) {  /* :40-61 */
  while (rc->range <= BOTTOM_VALUE) {
    if (rc->low < (0xFFu << SHIFT_BITS)) {
      TRC(tr_put(0); if (rc->help) TRB->help_nocarry++; if (TRB->help_in && !TRB->resolved_in) TRB->resolved_in = 1);
      put(rc->out, rc->buffer);
      for (; rc->help; rc->help--) put(rc->out, 0xFF);
      rc->buffer = (rc->low >> SHIFT_BITS) & 0xFF;
    } else if (rc->low & TOP_VALUE) {
      TRC(tr_put(1); TRB->carries++; if (rc->help) TRB->help_carry++; if (TRB->help_in && !TRB->resolved_in) TRB->resolved_in = 2);
      put(rc->out, rc->buffer + 1);
      for (; rc->help; rc->help--) put(rc->out, 0x00);
      rc->buffer = (rc->low >> SHIFT_BITS) & 0xFF;
    } else {
      rc->help++;
      TRC(if (rc->help > TRB->max_help) TRB->max_help = (uint32_t)rc->help;
          if (rc->help > TRF->max_help) TRF->max_help = (uint32_t)rc->help);
    }
    rc->range <<= 8;
    rc->low = (rc->low << 8) & (TOP_VALUE - 1);
    rc->bytecount++;
  }
}
static void enc_freq(rc_t* rc, uint32_t sy_f, uint32_t lt_f, uint32_t tot_f) {  /* :81-91 */
  enc_normalize(rc);
  TRC(tr_tot(rc->range, tot_f));
  const uint32_t r = rc->range / tot_f;
  const uint32_t tmp = r * lt_f;
  rc->low += tmp;
  if (lt_f + sy_f < tot_f) rc->range = r * sy_f; else rc->range -= tmp;
}
static void enc_shift(rc_t* rc, uint32_t sy_f, uint32_t lt_f, uint32_t shift) {  /* :92-102 */
  enc_normalize(rc);
  TRC(tr_tot(rc->range, 1u << shift));
  const uint32_t r = rc->range >> shift;
  const uint32_t tmp = r * lt_f;
  rc->low += tmp;
  if ((lt_f + sy_f) >> shift) rc->range -= tmp; else rc->range = r * sy_f;
}
static void enc_bit(rc_t* rc, uint32_t b) { enc_shift(rc, 1, b ? 1 : 0, 1); }   /* :104-106 */
static void enc_byte(rc_t* rc, uint32_t b) { enc_shift(rc, 1, b, 8); }          /* :108-110 */
static void enc_finish(rc_t* rc) {  /* :118-144 */
  enc_normalize(rc);
  rc->bytecount += 5;
  uint32_t tmp = rc->low >> SHIFT_BITS;
  if ((rc->low & (BOTTOM_VALUE - 1)) >= ((rc->bytecount & 0xFFFFFF) >> 1)) { tmp++; TRC(TRF->finish_round = 1); }
  TRC(TRF->finish_carry = tmp > 0xFF; TRF->bytecount = rc->bytecount; tr_put(tmp > 0xFF));
  if (tmp > 0xFF) {
    put(rc->out, rc->buffer + 1);
    for (; rc->help; rc->help--) put(rc->out, 0x00);
  } else {
    put(rc->out, rc->buffer);
    for (; rc->help; rc->help--) put(rc->out, 0xFF);
  }
  put(rc->out, tmp & 0xFF);
  put(rc->out, (rc->bytecount >> 16) & 0xFF);
  put(rc->out, (rc->bytecount >> 8) & 0xFF);
  put(rc->out, rc->bytecount & 0xFF);
}

static void dec_start_skipping_initial_read(rc_t* rc, src_t* in) {  /* :150-159 with skipInitialRead */
  rc->in = in; rc->out = NULL; rc->help = 0; rc->bytecount = 0;
  rc->buffer = (uint32_t)get(in);
  rc->low = rc->buffer >> (8 - EXTRA_BITS);
  rc->range = 1u << EXTRA_BITS;
}
static void dec_normalize(rc_t* rc) {  /* :161-170 */
  while (rc->range <= BOTTOM_VALUE) {
    rc->low = (rc->low << 8) | ((rc->buffer << EXTRA_BITS) & 0xFF);
    rc->buffer = (uint32_t)get(rc->in);   /* EOF reads as -1: all ones, like the reference's ToInt32(-1) */
    rc->low |= rc->buffer >> (8 - EXTRA_BITS);
    rc->range <<= 8;
  }
}
static uint32_t dec_culfreq(rc_t* rc, uint32_t tot_f) {  /* :177-182 */
  dec_normalize(rc);
  rc->help = rc->range / tot_f;
  const uint32_t tmp = (uint32_t)(rc->low / (uint32_t)rc->help);
  return tmp >= tot_f ? tot_f - 1 : tmp;
}
static uint32_t dec_culshift(rc_t* rc, uint32_t shift) {  /* :183-189 */
  dec_normalize(rc);
  rc->help = rc->range >> shift;
  const uint32_t tmp = (uint32_t)(rc->low / (uint32_t)rc->help);
  return (tmp >> shift) ? (1u << shift) - 1 : tmp;
}
static void dec_update(rc_t* rc, uint32_t sy_f, uint32_t lt_f, uint32_t tot_f) {  /* :197-205 */
  const uint32_t tmp = (uint32_t)rc->help * lt_f;
  rc->low -= tmp;
  if (lt_f + sy_f < tot_f) rc->range = (uint32_t)rc->help * sy_f; else rc->range -= tmp;
}
static uint32_t dec_bit(rc_t* rc) { uint32_t t = dec_culshift(rc, 1); dec_update(rc, 1, t, 2); return t; }      /* :208-212 */
static uint32_t dec_byte(rc_t* rc) { uint32_t t = dec_culshift(rc, 8); dec_update(rc, 1, t, 256); return t; }   /* :214-218 */

/* ---- NoModel over the range coder + LogDistanceModel ----------------------------------------------- */
static void raw_encode(rc_t* rc, int bits, uint32_t symbol) {  /* NoModel.js:15-21 */
  for (int i = bits - 1; i >= 0; i--) enc_bit(rc, (symbol >> i) & 1);
}
static uint32_t raw_decode(rc_t* rc, int bits) {  /* NoModel.js:22-29 */
  uint32_t r = 0;
  for (int i = bits - 1; i >= 0; i--) { r <<= 1; if (dec_bit(rc)) r++; }
  return r;
}
typedef struct { int lgbits; } logdist_t;  /* LogDistanceModel.js:8-23: lgDistanceModel = NoModel(1 + fls(size-1)) */
static void logdist_init(logdist_t* m, uint32_t size) { m->lgbits = fls32((uint32_t)(1 + fls32(size - 1)) - 1); }
static void logdist_encode(logdist_t* m, rc_t* rc, uint32_t distance) {  /* :26-39 */
  if (distance < 2) { raw_encode(rc, m->lgbits, distance); return; }
  const int lg = fls32(distance);
  raw_encode(rc, m->lgbits, (uint32_t)lg);
  raw_encode(rc, lg - 1, distance & ((1u << (lg - 1)) - 1));   /* distanceModel[lg] = NoModel(1 << (lg-1)): lg-1 bits */
}
static uint32_t logdist_decode(logdist_t* m, rc_t* rc) {  /* :40-47 */
  const uint32_t lg = raw_decode(rc, m->lgbits);
  if (lg < 2) return lg;
  if (lg > 31) return 0xffffffffu;
  return (1u << (lg - 1)) + raw_decode(rc, (int)lg - 1);
}

/* ---- FenwickModel (FenwickModel.js) --------------------------------------------------------------- */
#define ESC_MASK 0x0000FFFFu
#define SYM_MASK 0xFFFF0000u
#define SCALE_MASK 0xFFFEFFFEu
typedef struct { uint32_t numSyms, increment, max_prob; uint32_t tree[2 * 260]; rc_t* rc; } fen_t;

static void fen_sum(fen_t* f) {  /* :155-161 */
  for (uint32_t i = f->numSyms - 1; i > 0; i--) f->tree[i] = f->tree[2 * i] + f->tree[2 * i + 1];
}
static void fen_init(fen_t* f, rc_t* rc, uint32_t size, uint32_t max_prob, uint32_t increment) {  /* :15-33 */
  f->rc = rc; f->numSyms = size + 1; f->increment = increment; f->max_prob = max_prob;
  memset(f->tree, 0, sizeof f->tree);
  uint32_t i;
  for (i = 0; i < size; i++) f->tree[f->numSyms + i] = 1;          /* escape prob 1, symbol prob 0 */
  f->tree[f->numSyms + i] = increment << 16;                          /* the escape symbol itself */
  fen_sum(f);
}
static void fen_rescale(fen_t* f) {  /* :125-154 */
  uint32_t i, prob; int noEscape = 1;
  for (i = 0; i < f->numSyms - 1; i++) {
    prob = f->tree[f->numSyms + i];
    if (prob & ESC_MASK) { noEscape = 0; continue; }
    prob = (prob & SCALE_MASK) >> 1;
    if (prob == 0) { prob = 1; noEscape = 0; }
    f->tree[f->numSyms + i] = prob;
  }
  TRC(TRB->rescales++; TRB->rescales_noesc += noEscape);
  prob = f->tree[f->numSyms + i];
  prob = (prob & SCALE_MASK) >> 1;
  if (noEscape) prob = 0; else if (prob == 0) prob = 1u << 16;
  f->tree[f->numSyms + i] = prob;
  fen_sum(f);
}
static void fen_encode(fen_t* f, uint32_t symbol) {  /* :47-87 */
  uint32_t i = f->numSyms + symbol;
  uint32_t sy_f = f->tree[i];
  uint32_t mask = SYM_MASK, shift = 16;
  uint32_t update = f->increment << 16;
  if ((sy_f & SYM_MASK) == 0) {                       /* not seen yet: escape first, then code it among the unseen */
    TRC(TRB->escapes++; TRB->reescapes += TR_SEEN[symbol]; TR_SEEN[symbol] = 1; TRB->esc_lane31 += (TRB->nsym - 1) % 32 == 31);
    fen_encode(f, f->numSyms - 1);
    mask = ESC_MASK; update -= 1; shift = 0;
  } else if (symbol == f->numSyms - 1 && (f->tree[1] & ESC_MASK) == 1) {
    update = 0u - f->tree[i];                          /* the last escape: zero it out */
    TRC(TRB->last_escape++);
  }
  uint32_t lt_f = 0;
  while (i > 1) {
    const uint32_t parent = i >> 1;
    if (i & 1) lt_f += f->tree[2 * parent];
    f->tree[i] += update;
    i = parent;
  }
  uint32_t tot_f = f->tree[1];
  f->tree[1] += update;
  sy_f = (sy_f & mask) >> shift;
  lt_f = (lt_f & mask) >> shift;
  tot_f = (tot_f & mask) >> shift;
  enc_freq(f->rc, sy_f, lt_f, tot_f);
  TRC(if (((f->tree[1] & SYM_MASK) >> 16) >= f->max_prob) {
        TRB->rescales_esc += symbol == f->numSyms - 1;
        TRB->rescales_ff00 += ((f->tree[1] & SYM_MASK) >> 16) == f->max_prob; });
  if (((f->tree[1] & SYM_MASK) >> 16) >= f->max_prob) fen_rescale(f);
}
static uint32_t fen_decode1(fen_t* f, int isEscape) {  /* :88-123 */
  uint32_t mask = SYM_MASK, shift = 16;
  uint32_t update = f->increment << 16;
  if (isEscape) { mask = ESC_MASK; update -= 1; shift = 0; }
  const uint32_t tot_f = (f->tree[1] & mask) >> shift;
  if (tot_f == 0) return 0xffffffffu;                 /* corrupt stream: the reference would divide by zero */
  const uint32_t prob = dec_culfreq(f->rc, tot_f);
  uint32_t i = 1, lt_f = 0;
  while (i < f->numSyms) {
    f->tree[i] += update;
    const uint32_t leftProb = (f->tree[2 * i] & mask) >> shift;
    i *= 2;
    if (prob - lt_f >= leftProb) { lt_f += leftProb; i++; }
  }
  const uint32_t symbol = i - f->numSyms;
  const uint32_t sy_f = (f->tree[i] & mask) >> shift;
  f->tree[i] += update;
  dec_update(f->rc, sy_f, lt_f, tot_f);
  if (symbol == f->numSyms - 1 && (f->tree[1] & ESC_MASK) == 1) {
    update = 0u - f->tree[i];
    while (i >= 1) { f->tree[i] += update; i >>= 1; }
  }
  if (((f->tree[1] & SYM_MASK) >> 16) >= f->max_prob) fen_rescale(f);
  return symbol;
}
static uint32_t fen_decode(fen_t* f) {  /* :115-122 */
  uint32_t s = fen_decode1(f, 0);
  if (s == f->numSyms - 1) s = fen_decode1(f, 1);
  return s;
}

/* ---- DefSumModel (DefSumModel.js): deferred-sum model of the "fast" levels 1..5 ------------------------------ */
#define DS_LOG_TOTAL 8
#define DS_TOTAL 256u
#define DS_MAX_ESCAPE 40
typedef struct { uint32_t numSyms, updateCount, updateThresh; uint16_t prob[262], escape[262], update[262]; rc_t* rc; } dsm_t;

static void dsm_init(dsm_t* m, rc_t* rc, uint32_t size) {  /* :11-35 */
  memset(m, 0, sizeof *m);
  m->rc = rc; m->numSyms = size;
  m->prob[size + 1] = DS_TOTAL;                        /* everything escapes at first */
  for (uint32_t i = 0; i <= size; i++) m->escape[i] = (uint16_t)i;
  m->updateCount = 0;
  m->updateThresh = DS_TOTAL - DS_TOTAL / 2;
}
static void dsm_update(dsm_t* m, uint32_t symbol) {  /* :39-93 (the decoder's lookup tables are searched instead) */
  if (symbol == m->numSyms) {
    if (m->update[symbol] >= DS_MAX_ESCAPE) { TRC(TRB->ds_esc_cap++); return; }
    if (m->updateCount >= m->updateThresh - 1) return;   /* an escape never triggers the table rebuild */
  }
  m->update[symbol]++;
  m->updateCount++;
  if (m->updateCount < m->updateThresh) return;
  TRC(TRB->ds_rebuilds++);
  uint32_t cumProb = 0, cumEscProb = 0, odd = 0, i;
  m->escape[0] = 0; m->prob[0] = 0;
  for (i = 0; i < m->numSyms + 1; i++) {
    const uint32_t newProb = ((uint32_t)(m->prob[i + 1] - m->prob[i]) >> 1) + m->update[i];
    m->prob[i] = (uint16_t)cumProb;
    m->escape[i] = (uint16_t)cumEscProb;
    if (newProb) { cumProb += newProb; if (newProb & 1) odd++; }
    else cumEscProb++;
  }
  m->prob[i] = (uint16_t)cumProb;
  m->updateThresh = DS_TOTAL - (cumProb - odd) / 2;
  for (i = 0; i < m->numSyms + 1; i++) m->update[i] = 0;
  m->update[m->numSyms] = 1;
  m->updateCount = 1;
}
static void dsm_encode(dsm_t* m, uint32_t symbol) {  /* :94-111 */
  uint32_t lt_f = m->prob[symbol], sy_f = m->prob[symbol + 1] - lt_f;
  if (sy_f) { enc_shift(m->rc, sy_f, lt_f, DS_LOG_TOTAL); dsm_update(m, symbol); return; }
  TRC(TRB->escapes++; TRB->reescapes += TR_SEEN[symbol]; TR_SEEN[symbol] = 1; TRB->esc_lane31 += (TRB->nsym - 1) % 32 == 31);
  dsm_encode(m, m->numSyms);                            /* escape, then the symbol among the escaping ones */
  lt_f = m->escape[symbol];
  sy_f = m->escape[symbol + 1] - lt_f;
  enc_freq(m->rc, sy_f, lt_f, m->escape[m->numSyms]);
  dsm_update(m, symbol);
}
static uint32_t dsm_decode(dsm_t* m) {  /* :112-131 */
  uint32_t prob = dec_culshift(m->rc, DS_LOG_TOTAL), symbol = 0;
  while (symbol < m->numSyms && !(m->prob[symbol] <= prob && prob < m->prob[symbol + 1])) symbol++;   /* probToSym */
  uint32_t lt_f = m->prob[symbol], sy_f = m->prob[symbol + 1] - lt_f;
  dec_update(m->rc, sy_f, lt_f, DS_TOTAL);
  dsm_update(m, symbol);
  if (symbol != m->numSyms) return symbol;
  const uint32_t tot_f = m->escape[m->numSyms];
  if (tot_f == 0) return 0xffffffffu;
  prob = dec_culfreq(m->rc, tot_f);
  symbol = 0;
  while (symbol + 1 < m->numSyms && !(m->escape[symbol] <= prob && prob < m->escape[symbol + 1])) symbol++;   /* escProbToSym */
  lt_f = m->escape[symbol];
  sy_f = m->escape[symbol + 1] - lt_f;
  dec_update(m->rc, sy_f, lt_f, tot_f);
  dsm_update(m, symbol);
  return symbol;
}

/* ---- container ---------------------------------------------------------------------------------- */
#define F_PROB_MAX 0xFF00u   /* BWTC.js:7 */
#define F_PROB_INCR 0x0100u  /* BWTC.js:8 */

/* BWTC.compressFile(input, output, level) for a buffer input of known size (Util.js:105-141: the size is written).
 * With `blocks` (room for `cap` records) and `file`, also the trace of every block and of the file. */
static int bwtc_compress(const uint8_t* in, size_t n, int level, uint8_t** out, size_t* out_n, orc_bwtc_block_t* blocks,
                         size_t cap, orc_bwtc_file_t* file) {
  orc_bwtc_block_t scratch;
  memset(&scratch, 0, sizeof scratch);
  if (file) { memset(file, 0, sizeof *file); TRF = file; TRB = &scratch; }
  if (level < 1 || level > 9) level = 9;      /* BWTC.js:16-19: anything else means 9 */
  const int fast = level <= 5;                /* :22 */
  sink_t o = {0, 0, 0, 0};
  put(&o, 'b'); put(&o, 'w'); put(&o, 't'); put(&o, 'c');                      /* BWTC.js:11 */
  /* Util.js:194-209 writeUnsignedNumber(fileSize + 1), big endian 7-bit groups, last group flagged; the final byte
   * is handed to the range coder instead of being written (Util.js:125-132) */
  uint8_t grp[12]; int ng = 0;
  uint64_t v = (uint64_t)n + 1;
  do { grp[ng++] = (uint8_t)(v & 0x7F); v >>= 7; } while (v);
  grp[0] |= 0x80;
  for (int i = ng - 1; i >= 1; i--) put(&o, grp[i]);
  rc_t rc;
  enc_start(&rc, &o, grp[0], 1);                                                  /* BWTC.js:14 */
  enc_byte(&rc, (uint32_t)level);                                                 /* :21 */
  const uint32_t blockSize = (uint32_t)level * 100000u;                           /* :23 */
  uint8_t* U = (uint8_t*)malloc(blockSize ? blockSize : 1);
  fen_t* model = (fen_t*)malloc(sizeof(fen_t));
  dsm_t* dmodel = (dsm_t*)malloc(sizeof(dsm_t));
  if (!U || !model || !dmodel) { TRB = NULL; TRF = NULL; free(U); free(model); free(dmodel); free(o.p); return -6; }
  logdist_t lenModel;
  logdist_init(&lenModel, blockSize);                                             /* :40-42 */
  size_t pos = 0;
  uint32_t length;
  do {
    length = (uint32_t)((n - pos) < blockSize ? (n - pos) : blockSize);            /* readBlock :26-34 */
    if (length == 0) break;
    const uint8_t* b = in + pos;
    pos += length;
    if (file) {
      TRB = file->nblocks < cap ? &blocks[file->nblocks] : &scratch;
      memset(TRB, 0, sizeof *TRB);
      memset(TR_SEEN, 0, sizeof TR_SEEN);
      TRB->n = length;
      TRB->help_in = (uint32_t)rc.help;
      file->nblocks++;
    }
    if (length == blockSize) enc_freq(&rc, 1, 0, 3);                               /* :50-52 */
    else { enc_freq(&rc, 1, 1, 3); logdist_encode(&lenModel, &rc, length); }       /* :54-55 */
    const uint32_t pidx = (uint32_t)orc_bwt_sentinel(b, U, (int32_t)length);       /* :58 (returns pidx + 1) */
    logdist_encode(&lenModel, &rc, pidx);                                          /* :59 */
    uint16_t useTree[512];
    memset(useTree, 0, sizeof useTree);
    for (uint32_t i = 0; i < length; i++) useTree[256 + U[i]] = 1;                 /* :61-65 */
    for (int i = 255; i > 0; i--) useTree[i] = (uint16_t)(useTree[2 * i] + useTree[2 * i + 1]);
    useTree[0] = 1;
    for (uint32_t i = 1; i < 512; i++) {                                           /* :70-83 */
      const uint32_t parent = i >> 1, full = 1u << (9 - fls32(i));
      if (useTree[parent] == 0 || useTree[parent] == full * 2) continue;
      if (i >= 256) enc_bit(&rc, useTree[i]);
      else enc_freq(&rc, 1, useTree[i] == 0 ? 0u : (useTree[i] == full ? 2u : 1u), 3);
    }
    uint8_t M[256];
    uint32_t alphabetSize = 0;
    for (uint32_t i = 0; i < 256; i++) if (useTree[256 + i]) M[alphabetSize++] = (uint8_t)i;   /* :85-90 */
    TRC(TRB->alpha = alphabetSize);
    for (uint32_t i = 0; i < length; i++) {                                        /* :93-107 MTF */
      const uint8_t c = U[i];
      uint32_t j = 0;
      while (M[j] != c) j++;
      U[i] = (uint8_t)j;
      for (; j > 0; j--) M[j] = M[j - 1];
      M[0] = c;
    }
    if (fast) dsm_init(dmodel, &rc, alphabetSize + 1);                             /* :111 */
    else fen_init(model, &rc, alphabetSize + 1, F_PROB_MAX, F_PROB_INCR);          /* :109-110 */
#define MODEL_ENCODE(sym) do { TRC(TRB->nsym++); if (fast) dsm_encode(dmodel, (sym)); else fen_encode(model, (sym)); } while (0)
    uint32_t runLength = 0;
    for (uint32_t i = 0; i <= length; i++) {                                       /* :112-137; i == length flushes */
      const uint32_t c = i < length ? U[i] : 1u;
      if (i < length && c == 0) { runLength++; continue; }
      while (runLength) {                                                          /* emitLastRun :113-124 */
        if (runLength & 1) { MODEL_ENCODE(0); runLength -= 1; }
        else { MODEL_ENCODE(1); runLength -= 2; }
        runLength >>= 1;
      }
      if (i < length) MODEL_ENCODE(c + 1);
    }
#undef MODEL_ENCODE
    TRC(TRB->help = rc.help; TRB->bytes_out = o.n; TRB->bytecount = rc.bytecount; TRB = &scratch);
  } while (length == blockSize);                                                   /* :139 */
  enc_freq(&rc, 1, 2, 3);                                                           /* :141 */
  enc_finish(&rc);
  TRB = NULL; TRF = NULL;
  free(U); free(model); free(dmodel);
  if (o.oom) { free(o.p); return -6; }
  *out = o.p; *out_n = o.n;
  return 0;
}
ORC_EXPORT int orc_bwtc_compress(const uint8_t* in, size_t n, int level, uint8_t** out, size_t* out_n) {
  return bwtc_compress(in, n, level, out, out_n, NULL, 0, NULL);
}
ORC_EXPORT int orc_bwtc_compress_trace(const uint8_t* in, size_t n, int level, uint8_t** out, size_t* out_n,
                                       orc_bwtc_block_t* blocks, size_t cap, orc_bwtc_file_t* file) {
  return bwtc_compress(in, n, level, out, out_n, blocks, cap, file);
}

/* BWTC.decompressFile(input) (BWTC.js:141-231).  Returns 0, -2 for a bad magic ("Bad magic", Util.js:151-153),
 * -5 for a stream that decodes to nonsense (the reference has no checks: it would run off its buffers). */
ORC_EXPORT int orc_bwtc_decompress(const uint8_t* in, size_t n, uint8_t** out, size_t* out_n) {
  src_t s = {in, n, 0};
  if (get(&s) != 'b' || get(&s) != 'w' || get(&s) != 't' || get(&s) != 'c') return -2;
  /* Util.js:211-220 readUnsignedNumber; its last byte doubles as the range coder's first byte */
  uint64_t fs = 0;
  for (;;) {
    const int c = get(&s);
    if (c < 0) return -5;
    if (c & 0x80) { fs += (uint64_t)(c & 0x7F); break; }
    fs = (fs + (uint64_t)c) * 128;
  }
  rc_t rc;
  dec_start_skipping_initial_read(&rc, &s);                                        /* BWTC.js:143 */
  const uint32_t level = dec_byte(&rc);                                            /* :144 */
  if (level < 1 || level > 9) return -5;                                           /* :145 asserts */
  const int fast = level <= 5;
  const uint32_t blockSize = level * 100000u;
  sink_t o = {0, 0, 0, 0};
  uint8_t* block = (uint8_t*)malloc(blockSize + 2);
  uint8_t* U = (uint8_t*)malloc(blockSize);
  fen_t* model = (fen_t*)malloc(sizeof(fen_t));
  dsm_t* dmodel = (dsm_t*)malloc(sizeof(dsm_t));
  if (!block || !U || !model || !dmodel) { free(block); free(U); free(model); free(dmodel); return -6; }
  logdist_t lenModel;
  logdist_init(&lenModel, blockSize);
  int rcode = 0;
  for (;;) {
    const uint32_t ind = dec_culfreq(&rc, 3);                                      /* :158-159 */
    dec_update(&rc, 1, ind, 3);
    uint32_t length;
    if (ind == 0) length = blockSize;
    else if (ind == 1) length = logdist_decode(&lenModel, &rc);
    else break;
    if (length == 0 || length > blockSize) { rcode = -5; break; }
    const uint32_t pidx = logdist_decode(&lenModel, &rc);                          /* :170 */
    if (pidx > length) { rcode = -5; break; }
    uint16_t useTree[512];
    memset(useTree, 0, sizeof useTree);
    useTree[0] = 1;
    for (uint32_t i = 1; i < 512; i++) {                                           /* :172-187 */
      const uint32_t parent = i >> 1, full = 1u << (9 - fls32(i));
      if (useTree[parent] == 0 || useTree[parent] == full * 2) useTree[i] = useTree[parent] >> 1;
      else if (i >= 256) useTree[i] = (uint16_t)dec_bit(&rc);
      else { const uint32_t vv = dec_culfreq(&rc, 3); dec_update(&rc, 1, vv, 3); useTree[i] = (uint16_t)(vv == 2 ? full : vv); }
    }
    uint8_t M[256];
    uint32_t alphabetSize = 0;
    for (uint32_t i = 0; i < 256; i++) if (useTree[256 + i]) M[alphabetSize++] = (uint8_t)i;
    if (alphabetSize == 0) { rcode = -5; break; }
    if (fast) dsm_init(dmodel, &rc, alphabetSize + 1);                             /* :198 */
    else fen_init(model, &rc, alphabetSize + 1, F_PROB_MAX, F_PROB_INCR);          /* :196-197 */
    uint64_t val = 1;
    uint32_t i = 0;
    while (i < length) {                                                           /* :200-212 */
      const uint32_t c = fast ? dsm_decode(dmodel) : fen_decode(model);
      if (c == 0xffffffffu || c > alphabetSize) { rcode = -5; break; }
      if (c == 0 || c == 1) {
        const uint64_t cnt = val * (c + 1);
        if (cnt > length - i) { rcode = -5; break; }
        memset(block + i, 0, (size_t)cnt);
        i += (uint32_t)cnt;
        val *= 2;
      } else { val = 1; block[i++] = (uint8_t)(c - 1); }
    }
    if (rcode) break;
    for (i = 0; i < length; i++) {                                                 /* :214-222 inverse MTF */
      uint32_t j = block[i];
      if (j >= alphabetSize) { rcode = -5; break; }
      const uint8_t c = M[j];
      block[i] = c;
      for (; j > 0; j--) M[j] = M[j - 1];
      M[0] = c;
    }
    if (rcode) break;
    orc_unbwt_sentinel(block, U, (int32_t)length, (int32_t)pidx);                   /* :224 */
    for (i = 0; i < length; i++) put(&o, U[i]);
  }
  free(block); free(U); free(model); free(dmodel);
  if (!rcode && fs != 0 && o.n != fs - 1) rcode = -5;   /* Util.js:69-71: "outputsize does not match decoded input" */
  if (rcode || o.oom) { free(o.p); return rcode ? rcode : -6; }
  if (!o.p) o.p = (uint8_t*)malloc(1);
  *out = o.p; *out_n = o.n;
  return 0;
}
