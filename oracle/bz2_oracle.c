/*
 * oracle/bz2_oracle.c -- CPU restatement of the compressjs bzip2 block pipeline.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT THE PRODUCT.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load this library.  The
 * product path (compressjs_b200 -> libb2bz.so -> CUDA) never calls into it.
 *
 * Each function cites the reference file:line (under /root/reference) it restates.
 * The reference is JavaScript and cannot run in this image (no node); this file is a
 * plain-C restatement of its algorithm, pinned against the reference's own golden
 * vectors (test/bwtest.js KATs, test/huffman.js KATs, test/sample*.bz2 decode
 * fixtures, block extracts, .bzt tables) -- see tests/test_oracle_*.py.
 *
 * Declared engine semantics (SURVEY.md section 7): Array.prototype.sort at
 * lib/Bzip2.js:710 is STABLE (ES2019).  `legacy_sort` selects the pre-7.0 V8
 * insertion/quick sort instead, which reproduces the README.md:42,45 sizes.
 *
 * Encoder parity: pinned only by README sizes (legacy mode) -- the reference has no
 * golden compressed bytes (test/file.js is round-trip only).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <pthread.h>

#define ORC_EXPORT __attribute__((visibility("default")))

enum {
  ORC_OK = 0,
  ORC_LAST_BLOCK = -1,
  ORC_NOT_BZIP_DATA = -2,
  ORC_UNEXPECTED_INPUT_EOF = -3,
  ORC_UNEXPECTED_OUTPUT_EOF = -4,
  ORC_DATA_ERROR = -5,
  ORC_OUT_OF_MEMORY = -6,
  ORC_OBSOLETE_INPUT = -7,
  ORC_END_OF_BLOCK = -8
};

#define MAX_HUFCODE_BITS 20
#define MAX_SYMBOLS 258
#define GROUP_SIZE 50
#define MAX_GROUPS 6
#define MIN_GROUPS 2
static const uint64_t WHOLEPI = 0x314159265359ULL;
static const uint64_t SQRTPI = 0x177245385090ULL;

static __thread char g_err[256];
ORC_EXPORT const char* orc_last_error(void) { return g_err; }

/* ------------------------------------------------------------------ CRC32 */
/* lib/CRC32.js:37-103 -- MSB-first CRC-32/BZIP2, poly 0x04C11DB7. */
static uint32_t crc_tab[256];
static int crc_ready = 0;
static void crc_init(void) {
  if (crc_ready) return;
  for (uint32_t i = 0; i < 256; i++) {
    uint32_t c = i << 24;
    for (int k = 0; k < 8; k++) c = (c & 0x80000000u) ? (c << 1) ^ 0x04c11db7u : (c << 1);
    crc_tab[i] = c;
  }
  crc_ready = 1;
}
static inline uint32_t crc_update(uint32_t crc, uint8_t b) { /* CRC32.js:89-91 */
  return (crc << 8) ^ crc_tab[((crc >> 24) ^ b) & 0xff];
}
ORC_EXPORT uint32_t orc_crc32(const uint8_t* p, size_t n) {
  crc_init();
  uint32_t c = 0xffffffffu; /* CRC32.js:76 */
  for (size_t i = 0; i < n; i++) c = crc_update(c, p[i]);
  return ~c; /* CRC32.js:81-83 */
}

/* ------------------------------------------------------------ suffix sort */
/* Contract of lib/BWT.js:305-321 (suffixsort): plain suffix order, a proper prefix
 * sorts first.  The reference's SA-IS (BWT.js:21-300) is an implementation detail;
 * only its result is contractual.  This is prefix doubling (Manber-Myers with
 * counting sorts), O(n log n). */
static void suffix_sort(const uint8_t* T, int n, int* SA) {
  if (n <= 0) return;
  if (n == 1) { SA[0] = 0; return; }
  int m = n > 256 ? n : 256;
  int* rk = (int*)malloc(sizeof(int) * n);
  int* tmp = (int*)malloc(sizeof(int) * n);
  int* sa2 = (int*)malloc(sizeof(int) * n);
  int* cnt = (int*)calloc(m + 1, sizeof(int));
  for (int i = 0; i < n; i++) cnt[T[i]]++;
  for (int i = 1; i < 256; i++) cnt[i] += cnt[i - 1];
  for (int i = n - 1; i >= 0; i--) SA[--cnt[T[i]]] = i;
  int classes = 1;
  rk[SA[0]] = 0;
  for (int i = 1; i < n; i++) {
    if (T[SA[i]] != T[SA[i - 1]]) classes++;
    rk[SA[i]] = classes - 1;
  }
  for (int h = 1; classes < n; h <<= 1) {
    /* order by second key (rank of suffix i+h, "-1" when i+h >= n) */
    int p = 0;
    for (int i = (n - h > 0 ? n - h : 0); i < n; i++) sa2[p++] = i;
    for (int i = 0; i < n; i++) if (SA[i] >= h) sa2[p++] = SA[i] - h;
    /* stable counting sort by first key */
    memset(cnt, 0, sizeof(int) * (classes + 1));
    for (int i = 0; i < n; i++) cnt[rk[i]]++;
    for (int i = 1; i < classes; i++) cnt[i] += cnt[i - 1];
    for (int i = n - 1; i >= 0; i--) SA[--cnt[rk[sa2[i]]]] = sa2[i];
    /* new ranks */
    tmp[SA[0]] = 0;
    int nc = 1;
    for (int i = 1; i < n; i++) {
      int a = SA[i - 1], b = SA[i];
      int a2 = a + h < n ? rk[a + h] : -1, b2 = b + h < n ? rk[b + h] : -1;
      if (rk[a] != rk[b] || a2 != b2) nc++;
      tmp[b] = nc - 1;
    }
    int* t = rk; rk = tmp; tmp = t;
    classes = nc;
  }
  free(rk); free(tmp); free(sa2); free(cnt);
}

ORC_EXPORT int orc_suffixsort(const uint8_t* T, int32_t* SA, int32_t n) { /* BWT.js:305 */
  suffix_sort(T, n, SA);
  return 0;
}

/* lib/BWT.js:372-417 bwtransform2: CYCLIC BWT obtained by suffix-sorting the
 * doubled string TT=T+T and keeping the suffixes that start in the first half. */
ORC_EXPORT int32_t orc_bwt_cyclic(const uint8_t* T, uint8_t* U, int32_t n) {
  if (n <= 1) { if (n == 1) U[0] = T[0]; return 0; } /* BWT.js:376-379 */
  uint8_t* TT = (uint8_t*)malloc((size_t)2 * n);
  memcpy(TT, T, n); memcpy(TT + n, T, n); /* BWT.js:400-403 */
  int* A = (int*)malloc(sizeof(int) * 2 * (size_t)n);
  suffix_sort(TT, 2 * n, A); /* BWT.js:406 */
  int pidx = 0, j = 0;
  for (int i = 0; i < 2 * n; i++) { /* BWT.js:407-414 */
    int s = A[i];
    if (s < n) {
      if (s == 0) pidx = j;
      if (--s < 0) s = n - 1;
      U[j++] = T[s];
    }
  }
  free(TT); free(A);
  return pidx;
}

/* lib/BWT.js:328-350 bwtransform: sentinel (non-cyclic) BWT used by BWTC.
 * SA_IS(...,isbwt=true) (BWT.js:153-195 computeBWT) leaves in A the preceding
 * characters in suffix order, skipping suffix 0, and returns the rank slot of
 * suffix 0; U[0]=T[n-1]; returns pidx+1. */
ORC_EXPORT int32_t orc_bwt_sentinel(const uint8_t* T, uint8_t* U, int32_t n) {
  if (n <= 1) { if (n == 1) U[0] = T[0]; return n; }
  int* SA = (int*)malloc(sizeof(int) * (size_t)n);
  suffix_sort(T, n, SA);
  /* Output: U[0]=T[n-1] (char before the virtual sentinel suffix), then for each
   * suffix in order except suffix 0: T[s-1].  pidx = number of suffixes smaller
   * than suffix 0. */
  int pidx = 0, j = 1;
  U[0] = T[n - 1];
  for (int i = 0; i < n; i++) {
    int s = SA[i];
    if (s == 0) { pidx = i; continue; }
    U[j++] = T[s - 1];
  }
  free(SA);
  return pidx + 1;
}

/* lib/BWT.js:352-363 unbwtransform (inverse of the sentinel BWT). */
ORC_EXPORT int orc_unbwt_sentinel(const uint8_t* T, uint8_t* U, int32_t n, int32_t pidx) {
  uint32_t C[256];
  memset(C, 0, sizeof C);
  int32_t* LF = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
  for (int i = 0; i < n; i++) LF[i] = C[T[i]]++;
  uint32_t t = 0;
  for (int i = 0; i < 256; i++) { t += C[i]; C[i] = t - C[i]; }
  int32_t tt = 0;
  for (int i = n - 1; i >= 0; i--) {
    U[i] = T[tt];
    tt = LF[tt] + C[U[i]];
    tt += (tt < pidx) ? 1 : 0;
  }
  free(LF);
  return 0;
}

/* ------------------------------------------------------- HuffmanAllocator */
/* lib/HuffmanAllocator.js:52-75 first() */
static int ha_first(const int* array, int length, int i, int nodesToMove) {
  int limit = i;
  int k = length - 2;
  while ((i >= nodesToMove) && ((array[i] % length) > limit)) {
    k = i;
    i -= (limit - i + 1);
  }
  i = (nodesToMove - 1 > i) ? nodesToMove - 1 : i;
  while (k > (i + 1)) {
    int temp = (i + k) >> 1;
    if ((array[temp] % length) > limit) k = temp; else i = temp;
  }
  return k;
}
/* lib/HuffmanAllocator.js:79-105 */
static void ha_set_extended_parent_pointers(int* array, int length) {
  array[0] += array[1];
  int headNode, tailNode, topNode, temp;
  for (headNode = 0, tailNode = 1, topNode = 2; tailNode < (length - 1); tailNode++) {
    if ((topNode >= length) || (array[headNode] < array[topNode])) {
      temp = array[headNode];
      array[headNode++] = tailNode;
    } else {
      temp = array[topNode++];
    }
    if ((topNode >= length) || ((headNode < tailNode) && (array[headNode] < array[topNode]))) {
      temp += array[headNode];
      array[headNode++] = tailNode + length;
    } else {
      temp += array[topNode++];
    }
    array[tailNode] = temp;
  }
}
/* lib/HuffmanAllocator.js:114-124 */
static int ha_find_nodes_to_relocate(const int* array, int length, int maximumLength) {
  int currentNode = length - 2;
  for (int currentDepth = 1; (currentDepth < (maximumLength - 1)) && (currentNode > 1); currentDepth++)
    currentNode = ha_first(array, length, currentNode - 1, 0);
  return currentNode;
}
/* lib/HuffmanAllocator.js:131-148 */
static void ha_allocate_node_lengths(int* array, int length) {
  int firstNode = length - 2;
  int nextNode = length - 1;
  int currentDepth, availableNodes, lastNode, i;
  for (currentDepth = 1, availableNodes = 2; availableNodes > 0; currentDepth++) {
    lastNode = firstNode;
    firstNode = ha_first(array, length, lastNode - 1, 0);
    for (i = availableNodes - (lastNode - firstNode); i > 0; i--) array[nextNode--] = currentDepth;
    availableNodes = (lastNode - firstNode) << 1;
  }
}
/* lib/HuffmanAllocator.js:157-188 */
static void ha_allocate_node_lengths_with_relocation(int* array, int length, int nodesToMove, int insertDepth) {
  int firstNode = length - 2;
  int nextNode = length - 1;
  int currentDepth = (insertDepth == 1) ? 2 : 1;
  int nodesLeftToMove = (insertDepth == 1) ? nodesToMove - 2 : nodesToMove;
  int availableNodes, lastNode, offset, i;
  for (availableNodes = currentDepth << 1; availableNodes > 0; currentDepth++) {
    lastNode = firstNode;
    firstNode = (firstNode <= nodesToMove) ? firstNode : ha_first(array, length, lastNode - 1, nodesToMove);
    offset = 0;
    if (currentDepth >= insertDepth) {
      int cap = 1 << (currentDepth - insertDepth);
      offset = nodesLeftToMove < cap ? nodesLeftToMove : cap;
    } else if (currentDepth == (insertDepth - 1)) {
      offset = 1;
      if (array[firstNode] == lastNode) firstNode++;
    }
    for (i = availableNodes - (lastNode - firstNode + offset); i > 0; i--) array[nextNode--] = currentDepth;
    nodesLeftToMove -= offset;
    availableNodes = (lastNode - firstNode + offset) << 1;
  }
}
static int fls32(uint32_t v) { int r = 0; while (v) { r++; v >>= 1; } return r; } /* Util.js:298-314 */
/* lib/HuffmanAllocator.js:199-222 */
ORC_EXPORT void orc_huffman_code_lengths(int32_t* array, int32_t length, int32_t maximumLength) {
  switch (length) {
    case 2: array[1] = 1; /* fallthrough */
    case 1: array[0] = 1; return;
    case 0: return;
  }
  ha_set_extended_parent_pointers(array, length);
  int nodesToRelocate = ha_find_nodes_to_relocate(array, length, maximumLength);
  if ((array[0] % length) >= nodesToRelocate) {
    ha_allocate_node_lengths(array, length);
  } else {
    int insertDepth = maximumLength - fls32((uint32_t)(nodesToRelocate - 1));
    ha_allocate_node_lengths_with_relocation(array, length, nodesToRelocate, insertDepth);
  }
}

/* ----------------------------------------------------------- bit writer  */
/* lib/BitStream.js:52-59,68-73,93-105 + Util.js:53-78 (growable BufferStream). */
typedef struct { uint8_t* buf; size_t cap, len; uint32_t acc; int nacc; } bitw_t;
static void bw_init(bitw_t* w) { w->cap = 16384; w->buf = (uint8_t*)malloc(w->cap); w->len = 0; w->acc = 0; w->nacc = 0; }
static inline void bw_byte(bitw_t* w, uint8_t b) {
  if (w->len >= w->cap) { w->cap *= 2; w->buf = (uint8_t*)realloc(w->buf, w->cap); }
  w->buf[w->len++] = b;
}
static inline void bw_bits(bitw_t* w, int n, uint64_t v) { /* MSB first */
  for (int i = n - 1; i >= 0; i--) {
    w->acc = (w->acc << 1) | (uint32_t)((v >> i) & 1);
    if (++w->nacc == 8) { bw_byte(w, (uint8_t)w->acc); w->acc = 0; w->nacc = 0; }
  }
}
static inline void bw_flush(bitw_t* w) { while (w->nacc) bw_bits(w, 1, 0); } /* BitStream.js:68-73 */
static inline uint64_t bw_tellbit(const bitw_t* w) { return (uint64_t)w->len * 8 + w->nacc; }

/* ------------------------------------------------------ StaticHuffman    */
typedef struct { uint8_t len[MAX_SYMBOLS]; uint32_t code[MAX_SYMBOLS]; int n; } shuff_t;
static int cmp_int(const void* a, const void* b) { int x = *(const int*)a, y = *(const int*)b; return (x > y) - (x < y); }
/* lib/Bzip2.js:551-579 */
static void shuff_build(shuff_t* h, const int* freq, int alphabetSize) {
  int merged[MAX_SYMBOLS], sorted[MAX_SYMBOLS];
  for (int i = 0; i < alphabetSize; i++) merged[i] = (freq[i] << 9) | i;
  qsort(merged, alphabetSize, sizeof(int), cmp_int); /* keys are unique -> engine independent */
  for (int i = 0; i < alphabetSize; i++) sorted[i] = (int)((uint32_t)merged[i] >> 9);
  orc_huffman_code_lengths(sorted, alphabetSize, MAX_HUFCODE_BITS);
  h->n = alphabetSize;
  for (int i = 0; i < alphabetSize; i++) h->len[merged[i] & 0x1FF] = (uint8_t)sorted[i];
}
/* lib/Bzip2.js:581-600 */
static void shuff_canonical(shuff_t* h) {
  int merged[MAX_SYMBOLS];
  for (int i = 0; i < h->n; i++) merged[i] = (h->len[i] << 9) | i;
  qsort(merged, h->n, sizeof(int), cmp_int);
  uint32_t code = 0; int prevLen = 0;
  for (int i = 0; i < h->n; i++) {
    int curLen = merged[i] >> 9, sym = merged[i] & 0x1FF;
    code <<= (curLen - prevLen);
    h->code[sym] = code++;
    prevLen = curLen;
  }
}
/* lib/Bzip2.js:602-608 */
static inline int shuff_cost(const shuff_t* h, const uint16_t* a, int off, int len) {
  int c = 0;
  for (int i = 0; i < len; i++) c += h->len[a[off + i]];
  return c;
}
/* lib/Bzip2.js:610-629 */
static void shuff_emit(const shuff_t* h, bitw_t* w) {
  int cur = h->len[0];
  bw_bits(w, 5, cur);
  for (int i = 0; i < h->n; i++) {
    int cl = h->len[i], value, delta;
    if (cur < cl) { value = 2; delta = cl - cur; } else { value = 3; delta = cur - cl; }
    while (delta-- > 0) bw_bits(w, 2, value);
    bw_bits(w, 1, 0);
    cur = cl;
  }
}

/* lib/Bzip2.js:636-667 readBlock: RLE1 + CRC over the raw bytes consumed. */
static int read_block(const uint8_t* in, size_t n, size_t* ppos, uint8_t* block, int length, uint32_t* crc) {
  int pos = 0, lastChar = -1, runLength = 0;
  while (pos < length) {
    if (runLength == 4) {
      block[pos++] = 0;
      if (pos >= length) break;
    }
    if (*ppos >= n) break; /* EOF */
    int ch = in[(*ppos)++];
    *crc = crc_update(*crc, (uint8_t)ch);
    if (ch != lastChar) {
      lastChar = ch; runLength = 1;
    } else {
      runLength++;
      if (runLength > 4) {
        if (runLength < 256) { block[pos - 1]++; continue; }
        else runLength = 1;
      }
    }
    block[pos++] = (uint8_t)ch;
  }
  return pos;
}

/* lib/Bzip2.js:671-684 */
static void assign_selectors(uint8_t* selectors, shuff_t* groups, int ngroups, const uint16_t* input, int len) {
  for (int i = 0, k = 0; i < len; i += GROUP_SIZE) {
    int gs = len - i < GROUP_SIZE ? len - i : GROUP_SIZE;
    int best = 0, bestCost = shuff_cost(&groups[0], input, i, gs);
    for (int j = 1; j < ngroups; j++) {
      int c = shuff_cost(&groups[j], input, i, gs);
      if (c < bestCost) { best = j; bestCost = c; }
    }
    selectors[k++] = (uint8_t)best;
  }
}

typedef struct { int index, cost; } split_t;
static int cmp_split_stable(const void* a, const void* b) {
  const split_t* x = (const split_t*)a; const split_t* y = (const split_t*)b;
  if (x->cost != y->cost) return (x->cost > y->cost) - (x->cost < y->cost);
  return (x->index > y->index) - (x->index < y->index); /* stable: pushed in ascending index */
}
/* SURVEY.md Appendix A: legacy (pre-7.0) V8 Array.prototype.sort, comparator s1.cost-s2.cost. */
static inline int scmp(const split_t* a, const split_t* b) { return a->cost - b->cost; }
static void legacy_insertion(split_t* a, int from, int to) {
  for (int i = from + 1; i < to; i++) {
    split_t e = a[i]; int j;
    for (j = i - 1; j >= from; j--) {
      if (scmp(&a[j], &e) > 0) a[j + 1] = a[j]; else break;
    }
    a[j + 1] = e;
  }
}
static void legacy_quicksort(split_t* a, int from, int to) {
  for (;;) {
    if (to - from <= 10) { legacy_insertion(a, from, to); return; }
    int third = from + ((to - from) >> 1);
    split_t v0 = a[from], v1 = a[to - 1], v2 = a[third], t;
    int c01 = scmp(&v0, &v1);
    if (c01 > 0) { t = v0; v0 = v1; v1 = t; }
    int c02 = scmp(&v0, &v2);
    if (c02 >= 0) { t = v0; v0 = v2; v2 = v1; v1 = t; }
    else { int c12 = scmp(&v1, &v2); if (c12 > 0) { t = v1; v1 = v2; v2 = t; } }
    a[from] = v0; a[to - 1] = v2;
    split_t pivot = v1;
    int low_end = from + 1, high_start = to - 1;
    a[third] = a[low_end]; a[low_end] = pivot;
    for (int i = low_end + 1; i < high_start; i++) {
      split_t element = a[i];
      int order = scmp(&element, &pivot);
      if (order < 0) {
        a[i] = a[low_end]; a[low_end] = element; low_end++;
      } else if (order > 0) {
        int brk = 0;
        do {
          high_start--;
          if (high_start == i) { brk = 1; break; }
          order = scmp(&a[high_start], &pivot);
        } while (order > 0);
        if (brk) break;
        a[i] = a[high_start]; a[high_start] = element;
        if (order < 0) {
          element = a[i];
          a[i] = a[low_end]; a[low_end] = element; low_end++;
        }
      }
    }
    if (to - high_start < low_end - from) { legacy_quicksort(a, high_start, to); to = low_end; }
    else { legacy_quicksort(a, from, low_end); from = high_start; }
  }
}

/* lib/Bzip2.js:685-733 */
static void optimize_huffman_groups(shuff_t* groups, int* pngroups, int targetGroups, const uint16_t* input, int len,
                                    uint8_t* selectors, int nsel, int alphabetSize, int legacy_sort) {
  int ngroups = *pngroups;
  split_t* splits = (split_t*)malloc(sizeof(split_t) * (size_t)(nsel > 0 ? nsel : 1));
  int (*freq)[MAX_SYMBOLS] = (int (*)[MAX_SYMBOLS])malloc(sizeof(int) * MAX_SYMBOLS * MAX_GROUPS);
  while (ngroups < targetGroups) {
    assign_selectors(selectors, groups, ngroups, input, len);
    int groupCounts[MAX_GROUPS] = {0};
    for (int i = 0; i < nsel; i++) groupCounts[selectors[i]]++;
    int which = 0;
    for (int i = 1; i < ngroups; i++) if (groupCounts[i] > groupCounts[which]) which = i; /* indexOf(max) = first max */
    int ns = 0;
    for (int i = 0; i < nsel; i++) {
      if (selectors[i] != which) continue;
      int start = i * GROUP_SIZE;
      int end = start + GROUP_SIZE < len ? start + GROUP_SIZE : len;
      splits[ns].index = i;
      splits[ns].cost = shuff_cost(&groups[which], input, start, end - start);
      ns++;
    }
    if (legacy_sort) legacy_quicksort(splits, 0, ns);
    else qsort(splits, ns, sizeof(split_t), cmp_split_stable);
    for (int i = ns >> 1; i < ns; i++) selectors[splits[i].index] = (uint8_t)ngroups;
    ngroups++;
    memset(freq, 0, sizeof(int) * MAX_SYMBOLS * MAX_GROUPS);
    for (int i = 0, j = 0; i < len;) {
      int* f = freq[selectors[j++]];
      for (int k = 0; k < GROUP_SIZE && i < len; k++) f[input[i++]]++;
    }
    for (int i = 0; i < ngroups; i++) shuff_build(&groups[i], freq[i], alphabetSize);
  }
  free(splits); free(freq);
  *pngroups = ngroups;
}

/* Per-block trace, so that tests can compare CUDA stages one at a time. */
typedef struct {
  int32_t n;        /* post-RLE1 length */
  int32_t pidx;
  int32_t m;        /* MTF/RLE2 symbol count incl. EOB */
  int32_t alpha;    /* distinct bytes */
  int32_t ngroups;
  int32_t nsel;
  uint32_t crc;
  uint32_t pad;
  uint64_t raw_start; /* offset of the block's first raw byte */
  uint64_t raw_len;
  uint64_t bit_start; /* bit offset of the block magic in the output */
  uint64_t bit_len;   /* bits from magic to end of block body */
} orc_block_trace_t;

/* lib/Bzip2.js:735-876 compressBlock.  If sym_out != NULL the MTF/RLE2 symbols are copied there. */
static void compress_block(const uint8_t* block, int length, bitw_t* w, int legacy_sort, orc_block_trace_t* tr,
                           uint16_t* sym_out, uint8_t* sel_out, uint8_t* len_out) {
  uint8_t* U = (uint8_t*)malloc((size_t)length + 1);
  int pidx = orc_bwt_cyclic(block, U, length);
  bw_bits(w, 1, 0);
  bw_bits(w, 24, (uint64_t)pidx);
  int used[256] = {0}, compact[16] = {0};
  for (int i = 0; i < length; i++) { used[block[i]] = 1; compact[block[i] >> 4] = 1; }
  for (int i = 0; i < 16; i++) bw_bits(w, 1, compact[i]);
  for (int i = 0; i < 16; i++) if (compact[i]) for (int j = 0; j < 16; j++) bw_bits(w, 1, used[(i << 4) | j]);
  int alphabetSize = 0;
  for (int i = 0; i < 256; i++) if (used[i]) alphabetSize++;
  uint16_t* A = (uint16_t*)malloc(sizeof(uint16_t) * ((size_t)length + 1));
  int endOfBlock = alphabetSize + 1;
  int freq[MAX_SYMBOLS] = {0};
  uint8_t M[256];
  for (int i = 0, j = 0; i < 256; i++) if (used[i]) M[j++] = (uint8_t)i;
  int pos = 0; uint32_t runLength = 0;
#define EMIT(c) do { A[pos++] = (uint16_t)(c); freq[(c)]++; } while (0)
#define EMIT_LAST_RUN() do { while (runLength != 0) { if (runLength & 1) { EMIT(0); runLength -= 1; } else { EMIT(1); runLength -= 2; } runLength >>= 1; } } while (0)
  for (int i = 0; i < length; i++) {
    uint8_t c = U[i];
    int j;
    for (j = 0; j < alphabetSize; j++) if (M[j] == c) break;
    for (int k = j; k > 0; k--) M[k] = M[k - 1]; /* mtf() Bzip2.js:53-60 */
    M[0] = c;
    if (j == 0) runLength++;
    else { EMIT_LAST_RUN(); EMIT(j + 1); runLength = 0; }
  }
  EMIT_LAST_RUN();
  EMIT(endOfBlock);
  int targetGroups;
  if (pos >= 2400) targetGroups = 6; else if (pos >= 1200) targetGroups = 5;
  else if (pos >= 600) targetGroups = 4; else if (pos >= 200) targetGroups = 3; else targetGroups = 2;
  shuff_t groups[MAX_GROUPS];
  int ngroups = 0;
  shuff_build(&groups[ngroups++], freq, endOfBlock + 1);
  for (int i = 0; i <= endOfBlock; i++) freq[i] = 1;
  shuff_build(&groups[ngroups++], freq, endOfBlock + 1);
  int nsel = (pos + GROUP_SIZE - 1) / GROUP_SIZE;
  uint8_t* selectors = (uint8_t*)calloc((size_t)nsel + 1, 1);
  optimize_huffman_groups(groups, &ngroups, targetGroups, A, pos, selectors, nsel, endOfBlock + 1, legacy_sort);
  assign_selectors(selectors, groups, ngroups, A, pos);
  bw_bits(w, 3, ngroups);
  bw_bits(w, 15, nsel);
  for (int i = 0; i < ngroups; i++) M[i] = (uint8_t)i;
  for (int i = 0; i < nsel; i++) {
    uint8_t s = selectors[i];
    int j;
    for (j = 0; j < ngroups; j++) if (M[j] == s) break;
    for (int k = j; k > 0; k--) M[k] = M[k - 1];
    M[0] = s;
    for (; j > 0; j--) bw_bits(w, 1, 1);
    bw_bits(w, 1, 0);
  }
  for (int i = 0; i < ngroups; i++) { shuff_emit(&groups[i], w); shuff_canonical(&groups[i]); }
  for (int i = 0, k = 0; i < pos;) {
    shuff_t* h = &groups[selectors[k++]];
    for (int j = 0; j < GROUP_SIZE && i < pos; j++) { int s = A[i++]; bw_bits(w, h->len[s], h->code[s]); }
  }
  if (tr) { tr->n = length; tr->pidx = pidx; tr->m = pos; tr->alpha = alphabetSize; tr->ngroups = ngroups; tr->nsel = nsel; }
  if (sym_out) memcpy(sym_out, A, sizeof(uint16_t) * (size_t)pos);
  if (sel_out) memcpy(sel_out, selectors, (size_t)nsel);
  if (len_out) for (int g = 0; g < ngroups; g++) memcpy(len_out + g * MAX_SYMBOLS, groups[g].len, (size_t)(endOfBlock + 1));
  free(U); free(A); free(selectors);
}

/* lib/Bzip2.js:879-929 compressFile.  trace (optional) receives up to trace_cap entries;
 * *ntrace is set to the number of blocks. */
ORC_EXPORT int orc_bzip2_compress_ex(const uint8_t* in, size_t n, int level, int legacy_sort, uint8_t** out, size_t* out_n,
                                     orc_block_trace_t* trace, size_t trace_cap, size_t* ntrace) {
  crc_init();
  if (level < 1 || level > 9) { snprintf(g_err, sizeof g_err, "Invalid block size multiplier"); return -100; }
  int blockSize = level * 100000 - 19; /* Bzip2.js:892-900 */
  bitw_t w; bw_init(&w);
  bw_bits(&w, 8, 'B'); bw_bits(&w, 8, 'Z'); bw_bits(&w, 8, 'h'); bw_bits(&w, 8, '0' + level);
  uint8_t* block = (uint8_t*)malloc((size_t)blockSize);
  uint32_t streamCRC = 0;
  size_t pos = 0, nb = 0;
  int length;
  do {
    uint32_t crc = 0xffffffffu;
    size_t start = pos;
    length = read_block(in, n, &pos, block, blockSize, &crc);
    if (length > 0) {
      crc = ~crc;
      streamCRC = ((streamCRC << 1) | (streamCRC >> 31)) ^ crc; /* Bzip2.js:917 */
      uint64_t b0 = bw_tellbit(&w);
      bw_bits(&w, 48, WHOLEPI);
      bw_bits(&w, 32, crc);
      orc_block_trace_t* tr = (trace && nb < trace_cap) ? &trace[nb] : NULL;
      compress_block(block, length, &w, legacy_sort, tr, NULL, NULL, NULL);
      if (tr) { tr->crc = crc; tr->raw_start = start; tr->raw_len = pos - start; tr->bit_start = b0; tr->bit_len = bw_tellbit(&w) - b0; }
      nb++;
    }
  } while (length == blockSize);
  bw_bits(&w, 48, SQRTPI);
  bw_bits(&w, 32, streamCRC);
  bw_flush(&w);
  free(block);
  *out = w.buf; *out_n = w.len;
  if (ntrace) *ntrace = nb;
  return 0;
}
ORC_EXPORT int orc_bzip2_compress(const uint8_t* in, size_t n, int level, uint8_t** out, size_t* out_n) {
  return orc_bzip2_compress_ex(in, n, level, 0, out, out_n, NULL, 0, NULL);
}

/* Stage helpers for kernel-by-kernel parity tests. */
/* RLE1 block split only: fills starts/lens/crcs (cap entries) and, if blocks != NULL, the
 * post-RLE1 bytes of block k at blocks + k*stride. Returns number of blocks. */
ORC_EXPORT size_t orc_rle1_split(const uint8_t* in, size_t n, int level, uint64_t* raw_starts, uint32_t* lens, uint32_t* crcs,
                                 size_t cap, uint8_t* blocks, size_t stride) {
  crc_init();
  int blockSize = level * 100000 - 19;
  uint8_t* block = (uint8_t*)malloc((size_t)blockSize);
  size_t pos = 0, nb = 0; int length;
  do {
    uint32_t crc = 0xffffffffu; size_t start = pos;
    length = read_block(in, n, &pos, block, blockSize, &crc);
    if (length > 0) {
      if (nb < cap) {
        if (raw_starts) raw_starts[nb] = start;
        if (lens) lens[nb] = (uint32_t)length;
        if (crcs) crcs[nb] = ~crc;
        if (blocks) memcpy(blocks + nb * stride, block, (size_t)length);
      }
      nb++;
    }
  } while (length == blockSize);
  free(block);
  return nb;
}
/* One block, all stages: block bytes (post-RLE1) -> symbols, selectors, code lengths, bits.
 * sym (cap n+1 u16), sel (cap ceil((n+1)/50)), lens (6*258 bytes).  Returns the block body bits in *out. */
ORC_EXPORT int orc_compress_block_stages(const uint8_t* block, int32_t n, int legacy_sort, orc_block_trace_t* tr, uint16_t* sym,
                                         uint8_t* sel, uint8_t* lens, uint8_t** out, size_t* out_bits) {
  crc_init();
  bitw_t w; bw_init(&w);
  compress_block(block, n, &w, legacy_sort, tr, sym, sel, lens);
  *out_bits = (size_t)bw_tellbit(&w);
  bw_flush(&w);
  *out = w.buf;
  return 0;
}

/* ------------------------------------------------------------- decoder   */
/* lib/BitStream.js:8-21,80-92 + Util.js:9-29: MSB-first reader; bits past EOF are zeros. */
typedef struct { const uint8_t* p; size_t n; size_t pos; uint32_t bufferByte; int eof_flag; } bitr_t;
static void br_init(bitr_t* r, const uint8_t* p, size_t n) { r->p = p; r->n = n; r->pos = 0; r->bufferByte = 0x100; r->eof_flag = 0; }
static inline int br_bit(bitr_t* r) {
  if ((r->bufferByte & 0xFF) == 0) {
    if (r->pos >= r->n) { r->eof_flag = 1; return 0; } /* EOF: reads as zero (BitStream.js:88-89) */
    r->bufferByte = ((uint32_t)r->p[r->pos++] << 1) | 1;
  }
  int bit = (r->bufferByte & 0x100) ? 1 : 0;
  r->bufferByte <<= 1;
  r->bufferByte &= 0x1FF;
  return bit;
}
static inline uint64_t br_bits(bitr_t* r, int n) { uint64_t v = 0; for (int i = 0; i < n; i++) v = (v << 1) | (uint64_t)br_bit(r); return v; }
static inline int br_stream_eof(const bitr_t* r) { return r->pos >= r->n; } /* Util.js:28 eof() of the byte stream */
static inline uint64_t br_tellbit(const bitr_t* r) { /* BitStream.js:29-37 */
  uint64_t pos = (uint64_t)r->pos * 8; uint32_t b = r->bufferByte;
  while ((b & 0xFF) != 0) { pos--; b = (b << 1) & 0x1FF; }
  return pos;
}
static inline void br_seekbit(bitr_t* r, uint64_t pos) { /* BitStream.js:22-28 */
  r->pos = (size_t)(pos >> 3); r->bufferByte = 0x100; r->eof_flag = 0;
  br_bits(r, (int)(pos & 7));
}

typedef struct { uint8_t* buf; size_t cap, len; } obuf_t;
static inline void ob_put(obuf_t* o, uint8_t b) {
  if (o->len >= o->cap) { o->cap = o->cap ? o->cap * 2 : 16384; o->buf = (uint8_t*)realloc(o->buf, o->cap); }
  o->buf[o->len++] = b;
}

typedef struct {
  bitr_t rd; int dbufSize; uint32_t streamCRC; uint32_t targetBlockCRC;
  uint32_t* dbuf; int writePos, writeCurrent, writeCount, writeRun;
} bunzip_t;

#define THROW(code, ...) do { snprintf(g_err, sizeof g_err, __VA_ARGS__); return (code); } while (0)

/* lib/Bzip2.js:105-124 */
static int start_bunzip(bunzip_t* bz) {
  uint8_t buf[4]; int got = 0;
  /* inputStream.read(buf,0,4) reads from the BYTE stream (resyncs the bit reader for multistream) */
  while (got < 4 && bz->rd.pos < bz->rd.n) buf[got++] = bz->rd.p[bz->rd.pos++];
  bz->rd.bufferByte = 0x100;
  if (got != 4 || buf[0] != 'B' || buf[1] != 'Z' || buf[2] != 'h') THROW(ORC_NOT_BZIP_DATA, "Not bzip data: bad magic");
  int level = buf[3] - 0x30;
  if (level < 1 || level > 9) THROW(ORC_NOT_BZIP_DATA, "Not bzip data: level out of range");
  bz->dbufSize = 100000 * level;
  bz->streamCRC = 0;
  return 0;
}

/* lib/Bzip2.js:125-398.  Returns 1 = block ready, 0 = end-of-stream marker seen, <0 = error. */
static int get_next_block(bunzip_t* bz) {
  bitr_t* reader = &bz->rd;
  uint64_t h = br_bits(reader, 48);
  if (h == SQRTPI) return 0;
  if (h != WHOLEPI) THROW(ORC_NOT_BZIP_DATA, "Not bzip data");
  bz->targetBlockCRC = (uint32_t)br_bits(reader, 32);
  bz->streamCRC = bz->targetBlockCRC ^ ((bz->streamCRC << 1) | (bz->streamCRC >> 31));
  if (br_bits(reader, 1)) THROW(ORC_OBSOLETE_INPUT, "Obsolete (pre 0.9.5) bzip format not supported.");
  int origPointer = (int)br_bits(reader, 24);
  if (origPointer > bz->dbufSize) THROW(ORC_DATA_ERROR, "Data error: initial position out of bounds");
  int t = (int)br_bits(reader, 16);
  uint8_t symToByte[256]; int symTotal = 0;
  memset(symToByte, 0, sizeof symToByte);
  for (int i = 0; i < 16; i++) {
    if (t & (1 << (0xF - i))) {
      int o = i * 16;
      int k = (int)br_bits(reader, 16);
      for (int j = 0; j < 16; j++) if (k & (1 << (0xF - j))) symToByte[symTotal++] = (uint8_t)(o + j);
    }
  }
  int groupCount = (int)br_bits(reader, 3);
  if (groupCount < MIN_GROUPS || groupCount > MAX_GROUPS) THROW(ORC_DATA_ERROR, "Data error");
  int nSelectors = (int)br_bits(reader, 15);
  if (nSelectors == 0) THROW(ORC_DATA_ERROR, "Data error");
  /* Util.makeU8Buffer(256) is zero-filled: a selector MTF index j == groupCount is legal and reads slot groupCount as 0 */
  uint8_t mtfSymbol[256];
  memset(mtfSymbol, 0, sizeof mtfSymbol);
  for (int i = 0; i < groupCount; i++) mtfSymbol[i] = (uint8_t)i;
  uint8_t* selectors = (uint8_t*)malloc((size_t)nSelectors);
  for (int i = 0; i < nSelectors; i++) {
    int j;
    for (j = 0; br_bits(reader, 1); j++) if (j >= groupCount) { free(selectors); THROW(ORC_DATA_ERROR, "Data error"); }
    uint8_t src = mtfSymbol[j];
    for (int k = j; k > 0; k--) mtfSymbol[k] = mtfSymbol[k - 1];
    mtfSymbol[0] = src;
    selectors[i] = src;
  }
  int symCount = symTotal + 2;
  struct { uint16_t permute[MAX_SYMBOLS]; int64_t limit[MAX_HUFCODE_BITS + 2]; int64_t base[MAX_HUFCODE_BITS + 1]; int minLen, maxLen; } groups[MAX_GROUPS];
  for (int j = 0; j < groupCount; j++) {
    uint8_t length[MAX_SYMBOLS]; uint16_t temp[MAX_HUFCODE_BITS + 1];
    memset(temp, 0, sizeof temp);
    t = (int)br_bits(reader, 5);
    for (int i = 0; i < symCount; i++) {
      for (;;) {
        if (t < 1 || t > MAX_HUFCODE_BITS) { free(selectors); THROW(ORC_DATA_ERROR, "Data error"); }
        if (!br_bits(reader, 1)) break;
        if (!br_bits(reader, 1)) t++; else t--;
      }
      length[i] = (uint8_t)t;
    }
    int minLen, maxLen;
    minLen = maxLen = length[0];
    for (int i = 1; i < symCount; i++) { if (length[i] > maxLen) maxLen = length[i]; else if (length[i] < minLen) minLen = length[i]; }
    memset(&groups[j], 0, sizeof groups[j]);
    groups[j].minLen = minLen; groups[j].maxLen = maxLen;
    int pp = 0;
    for (int i = minLen; i <= maxLen; i++) {
      temp[i] = 0; groups[j].limit[i] = 0;
      for (t = 0; t < symCount; t++) if (length[t] == i) groups[j].permute[pp++] = (uint16_t)t;
    }
    for (int i = 0; i < symCount; i++) temp[length[i]]++;
    pp = t = 0;
    for (int i = minLen; i < maxLen; i++) {
      pp += temp[i];
      groups[j].limit[i] = pp - 1;
      pp <<= 1;
      t += temp[i];
      groups[j].base[i + 1] = pp - t;
    }
    groups[j].limit[maxLen + 1] = INT64_MAX;
    groups[j].limit[maxLen] = pp + temp[maxLen] - 1;
    groups[j].base[minLen] = 0;
  }
  uint32_t byteCount[256];
  memset(byteCount, 0, sizeof byteCount);
  for (int i = 0; i < 256; i++) mtfSymbol[i] = (uint8_t)i;
  int runPos = 0, dbufCount = 0, selector = 0; uint8_t uc;
  free(bz->dbuf);
  uint32_t* dbuf = bz->dbuf = (uint32_t*)calloc((size_t)bz->dbufSize, sizeof(uint32_t));
  symCount = 0;
  int hg = 0; int64_t tt = 0;
  for (;;) {
    if (!(symCount--)) {
      symCount = GROUP_SIZE - 1;
      if (selector >= nSelectors) { free(selectors); THROW(ORC_DATA_ERROR, "Data error"); }
      hg = selectors[selector++];
    }
    int i = groups[hg].minLen;
    int64_t j = (int64_t)br_bits(reader, i);
    for (;; i++) {
      if (i > groups[hg].maxLen) { free(selectors); THROW(ORC_DATA_ERROR, "Data error"); }
      if (j <= groups[hg].limit[i]) break;
      j = (j << 1) | br_bits(reader, 1);
    }
    j -= groups[hg].base[i];
    if (j < 0 || j >= MAX_SYMBOLS) { free(selectors); THROW(ORC_DATA_ERROR, "Data error"); }
    int nextSym = groups[hg].permute[j];
    if (nextSym == 0 || nextSym == 1) {
      if (!runPos) { runPos = 1; tt = 0; }
      if (nextSym == 0) tt += runPos; else tt += 2 * (int64_t)runPos;
      runPos <<= 1;
      /* JS numbers do not overflow here; guard our int the way the later bound check would. */
      if (tt > (int64_t)bz->dbufSize * 4) { free(selectors); THROW(ORC_DATA_ERROR, "Data error"); }
      continue;
    }
    if (runPos) {
      runPos = 0;
      if (dbufCount + tt > bz->dbufSize) { free(selectors); THROW(ORC_DATA_ERROR, "Data error"); }
      uc = symToByte[mtfSymbol[0]];
      byteCount[uc] += (uint32_t)tt;
      while (tt--) dbuf[dbufCount++] = uc;
    }
    if (nextSym > symTotal) break;
    if (dbufCount >= bz->dbufSize) { free(selectors); THROW(ORC_DATA_ERROR, "Data error"); }
    i = nextSym - 1;
    uc = mtfSymbol[i];
    for (int k = i; k > 0; k--) mtfSymbol[k] = mtfSymbol[k - 1];
    mtfSymbol[0] = uc;
    uc = symToByte[uc];
    byteCount[uc]++;
    dbuf[dbufCount++] = uc;
  }
  free(selectors);
  if (origPointer < 0 || origPointer >= dbufCount) THROW(ORC_DATA_ERROR, "Data error");
  uint32_t jj = 0;
  for (int i = 0; i < 256; i++) { uint32_t k = jj + byteCount[i]; byteCount[i] = jj; jj = k; }
  for (int i = 0; i < dbufCount; i++) {
    uc = (uint8_t)(dbuf[i] & 0xff);
    dbuf[byteCount[uc]] |= ((uint32_t)i << 8);
    byteCount[uc]++;
  }
  int pos = 0, current = 0, run = 0;
  if (dbufCount) {
    pos = (int)dbuf[origPointer];
    current = pos & 0xff;
    pos = (int)((uint32_t)pos >> 8);
    run = -1;
  }
  bz->writePos = pos; bz->writeCurrent = current; bz->writeCount = dbufCount; bz->writeRun = run;
  return 1;
}

/* lib/Bzip2.js:405-448 */
static int read_bunzip(bunzip_t* bz, obuf_t* out) {
  if (bz->writeCount < 0) return 0;
  uint32_t* dbuf = bz->dbuf; int pos = bz->writePos, current = bz->writeCurrent, dbufCount = bz->writeCount, run = bz->writeRun;
  uint32_t crc = 0xffffffffu;
  while (dbufCount) {
    dbufCount--;
    int previous = current, copies, outbyte;
    uint32_t e = dbuf[pos];
    current = (int)(e & 0xff);
    pos = (int)(e >> 8);
    if (run++ == 3) { copies = current; outbyte = previous; current = -1; }
    else { copies = 1; outbyte = current; }
    while (copies--) { crc = crc_update(crc, (uint8_t)outbyte); ob_put(out, (uint8_t)outbyte); }
    if (current != previous) run = 0;
  }
  bz->writeCount = dbufCount;
  crc = ~crc;
  if (crc != bz->targetBlockCRC) THROW(ORC_DATA_ERROR, "Data error: Bad block CRC (got %x expected %x)", crc, bz->targetBlockCRC);
  return 0;
}

/* lib/Bzip2.js:454-481 Bunzip.decode.  If table_pos/table_len are given this behaves as
 * Bunzip.table (Bzip2.js:508-548): no stream-CRC check, records (bit position, bytes). */
static int decode_impl(const uint8_t* in, size_t n, int multistream, obuf_t* out, int as_table, uint64_t** tpos, uint32_t** tlen,
                       size_t* tcount) {
  crc_init();
  bunzip_t bz; memset(&bz, 0, sizeof bz);
  br_init(&bz.rd, in, n);
  int rc = start_bunzip(&bz);
  if (rc) return rc;
  size_t tc = 0, tcap = 0;
  for (;;) {
    if (br_stream_eof(&bz.rd)) break; /* Bzip2.js:462 / 527 */
    uint64_t position = br_tellbit(&bz.rd);
    rc = get_next_block(&bz);
    if (rc < 0) { free(bz.dbuf); return rc; }
    if (rc == 1) {
      size_t start = out->len;
      rc = read_bunzip(&bz, out);
      if (rc < 0) { free(bz.dbuf); return rc; }
      if (as_table) {
        if (tc >= tcap) { tcap = tcap ? tcap * 2 : 64; *tpos = (uint64_t*)realloc(*tpos, tcap * 8); *tlen = (uint32_t*)realloc(*tlen, tcap * 4); }
        (*tpos)[tc] = position; (*tlen)[tc] = (uint32_t)(out->len - start); tc++;
        out->len = 0; /* table() discards the bytes */
      }
    } else {
      uint32_t target = (uint32_t)br_bits(&bz.rd, 32);
      if (!as_table && target != bz.streamCRC) {
        free(bz.dbuf);
        THROW(ORC_DATA_ERROR, "Data error: Bad stream CRC (got %x expected %x)", bz.streamCRC, target);
      }
      if (multistream && !br_stream_eof(&bz.rd)) {
        rc = start_bunzip(&bz);
        if (rc) { free(bz.dbuf); return rc; }
      } else break;
    }
  }
  free(bz.dbuf);
  if (tcount) *tcount = tc;
  return 0;
}
ORC_EXPORT int orc_bzip2_decompress(const uint8_t* in, size_t n, int multistream, uint8_t** out, size_t* out_n) {
  obuf_t o = {0, 0, 0};
  int rc = decode_impl(in, n, multistream, &o, 0, NULL, NULL, NULL);
  if (rc) { free(o.buf); *out = NULL; *out_n = 0; return rc; }
  *out = o.buf ? o.buf : (uint8_t*)malloc(1); *out_n = o.len;
  return 0;
}
ORC_EXPORT int orc_bzip2_table(const uint8_t* in, size_t n, int multistream, uint64_t** bitpos, uint32_t** sizes, size_t* count) {
  obuf_t o = {0, 0, 0};
  *bitpos = NULL; *sizes = NULL; *count = 0;
  int rc = decode_impl(in, n, multistream, &o, 1, bitpos, sizes, count);
  free(o.buf);
  return rc;
}
/* lib/Bzip2.js:482-503 Bunzip.decodeBlock */
ORC_EXPORT int orc_bzip2_decompress_block(const uint8_t* in, size_t n, uint64_t bitpos, uint8_t** out, size_t* out_n) {
  crc_init();
  bunzip_t bz; memset(&bz, 0, sizeof bz);
  br_init(&bz.rd, in, n);
  int rc = start_bunzip(&bz);
  if (rc) return rc;
  br_seekbit(&bz.rd, bitpos);
  obuf_t o = {0, 0, 0};
  rc = get_next_block(&bz);
  if (rc < 0) { free(bz.dbuf); return rc; }
  if (rc == 1) {
    rc = read_bunzip(&bz, &o);
    if (rc < 0) { free(bz.dbuf); free(o.buf); return rc; }
  }
  free(bz.dbuf);
  *out = o.buf ? o.buf : (uint8_t*)malloc(1); *out_n = o.len;
  return 0;
}

ORC_EXPORT void orc_free(void* p) { free(p); }

/* --------------------------------------------- multi-threaded reference arm */
/* bench.py --impl reference: the same restated algorithm, blocks compressed by a pool of
 * host threads (the reference itself is single-threaded; this only lets the CPU arm use
 * every host core as the bench contract asks).  Output bytes are identical to
 * orc_bzip2_compress. */
typedef struct {
  const uint8_t* blocks; size_t stride; const uint32_t* lens; size_t nb; size_t next; pthread_mutex_t mu;
  uint8_t** bits; size_t* nbits;
} mt_job_t;
static void* mt_worker(void* arg) {
  mt_job_t* j = (mt_job_t*)arg;
  for (;;) {
    pthread_mutex_lock(&j->mu);
    size_t k = j->next++;
    pthread_mutex_unlock(&j->mu);
    if (k >= j->nb) break;
    bitw_t w; bw_init(&w);
    compress_block(j->blocks + k * j->stride, (int)j->lens[k], &w, 0, NULL, NULL, NULL, NULL);
    j->nbits[k] = (size_t)bw_tellbit(&w);
    bw_flush(&w);
    j->bits[k] = w.buf;
  }
  return NULL;
}
ORC_EXPORT int orc_bzip2_compress_mt(const uint8_t* in, size_t n, int level, int threads, uint8_t** out, size_t* out_n) {
  crc_init();
  if (level < 1 || level > 9) return -100;
  size_t stride = (size_t)level * 100000;
  /* a block holds at least 4/5 of blockSize raw bytes (runs of exactly four: 5 RLE1 bytes per 4 raw bytes) */
  size_t cap = n / ((size_t)(level * 100000 - 19) * 4 / 5) + 2;
  uint64_t* starts = (uint64_t*)malloc(8 * cap); uint32_t* lens = (uint32_t*)malloc(4 * cap); uint32_t* crcs = (uint32_t*)malloc(4 * cap);
  uint8_t* blocks = (uint8_t*)malloc(stride * cap);
  size_t nb = orc_rle1_split(in, n, level, starts, lens, crcs, cap, blocks, stride);
  if (nb > cap) { /* the split kept only `cap` blocks: fail rather than compress a truncated list */
    free(starts); free(lens); free(crcs); free(blocks);
    return -101;
  }
  mt_job_t job; job.blocks = blocks; job.stride = stride; job.lens = lens; job.nb = nb; job.next = 0;
  pthread_mutex_init(&job.mu, NULL);
  job.bits = (uint8_t**)calloc(nb + 1, sizeof(uint8_t*)); job.nbits = (size_t*)calloc(nb + 1, sizeof(size_t));
  if (threads < 1) threads = 1;
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)threads);
  for (int t = 0; t < threads; t++) pthread_create(&th[t], NULL, mt_worker, &job);
  for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
  bitw_t w; bw_init(&w);
  bw_bits(&w, 8, 'B'); bw_bits(&w, 8, 'Z'); bw_bits(&w, 8, 'h'); bw_bits(&w, 8, '0' + level);
  uint32_t streamCRC = 0;
  for (size_t k = 0; k < nb; k++) {
    streamCRC = ((streamCRC << 1) | (streamCRC >> 31)) ^ crcs[k];
    bw_bits(&w, 48, WHOLEPI); bw_bits(&w, 32, crcs[k]);
    size_t nbit = job.nbits[k]; const uint8_t* b = job.bits[k];
    size_t full = nbit >> 3;
    for (size_t i = 0; i < full; i++) bw_bits(&w, 8, b[i]);
    int rem = (int)(nbit & 7);
    if (rem) bw_bits(&w, rem, b[full] >> (8 - rem));
    free(job.bits[k]);
  }
  bw_bits(&w, 48, SQRTPI); bw_bits(&w, 32, streamCRC); bw_flush(&w);
  free(job.bits); free(job.nbits); free(th); free(starts); free(lens); free(crcs); free(blocks);
  pthread_mutex_destroy(&job.mu);
  *out = w.buf; *out_n = w.len;
  return 0;
}
