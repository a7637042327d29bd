/* TEST INFRASTRUCTURE ONLY -- never on the product path.
 *
 * Plain-C CPU restatement of the FastGA seed-and-extend hot path, used as the parity oracle for
 * the CUDA kernels in fastga_b200/csrc.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline leg may load this library.
 *
 * Pinned (tests/test_oracle_pin.py) against the UNMODIFIED reference compiled into oracle/_ref:
 *   - orc_local_alignment   vs  Local_Alignment of libfastga_ref.so (align.c:1423) on the same
 *                               sequences / tubes, Path + trace bytes bit-exact
 *   - orc_gix_build         vs  the .gix/.ktab files written by oracle/_ref/GIXmake
 *   - orc_merge + orc_search vs the .1aln written by oracle/_ref/FastGA (through ONEview); orc_chains
 *                               lists the chains of orc_search's own scan (one function serves both)
 *
 * Each function cites the reference lines it restates.  It is a restatement, not a copy: the two
 * wave routines of align.c are folded into one direction-normalised routine, M is derived from T
 * by popcount, the REACH/"more*" bookkeeping that FastGA never enables (reach = 0,
 * FastGA.c:3760) is dropped, and the merge works on 128-bit records instead of byte streams.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include <limits.h>

typedef struct { uint64_t lo, hi; } rec128;     /* same layout as fastga_b200/csrc/common.cuh */

#define KMER 40

/***********************************************************************************************
 *  A.  GIX construction: syncmer scan (GIXmake.c:406-611), record build (:802-980), sort
 *      (MSDsort.c), prefix index (GIXmake.c:1211-1278).
 **********************************************************************************************/

static const uint8_t TMap[256] =      /* GIXmake.c:92-109 -- hash definition, must be identical */
  { 0xff,0xd4,0xf5,0xfd,0xe4,0xad,0x21,0xa5,0xed,0x64,0xbf,0xa9,0xf3,0x70,0xd6,0xf0,
    0xca,0x89,0xcb,0xc9,0x82,0x9d,0x13,0x79,0x0a,0x0f,0x25,0x19,0x3e,0x47,0xa3,0xa8,
    0xf9,0x5e,0xe8,0xa1,0xb0,0x71,0x1d,0x8c,0xde,0x69,0xe7,0x7c,0x56,0x3f,0x90,0xa4,
    0xeb,0x45,0x59,0xf1,0x97,0x4c,0x08,0xa0,0xb8,0x4a,0x86,0xc8,0xcd,0x98,0x7d,0xfc,
    0xef,0x4d,0x83,0x7e,0xdc,0x66,0x2b,0x8e,0xe0,0xa7,0xd0,0xa2,0x88,0x5f,0x7f,0xd9,
    0x9b,0x78,0xd1,0x8b,0xc3,0x8f,0x2d,0xe6,0x18,0x27,0x2c,0x24,0x94,0xb7,0xce,0xbd,
    0x0d,0x04,0x1c,0x09,0x16,0x23,0x00,0x1e,0x1a,0x29,0x2e,0x15,0x01,0x10,0x2a,0x20,
    0xbe,0x31,0x43,0x58,0xc2,0xaa,0x1f,0xe5,0xc5,0x9e,0xcf,0xc6,0x68,0xb2,0x80,0xf4,
    0xf8,0x53,0xb6,0x93,0x76,0x37,0x11,0x40,0xda,0x51,0xba,0x46,0x42,0x30,0x60,0x6d,
    0x5c,0x39,0x9f,0x48,0x6c,0x62,0x28,0x67,0x06,0x12,0x26,0x0e,0x33,0x50,0xa6,0x63,
    0xdd,0x3b,0xab,0x4b,0x72,0x5b,0x22,0x6f,0xb4,0x61,0x92,0x99,0x36,0x38,0x65,0xac,
    0x4f,0x2f,0x32,0x44,0x54,0x3c,0x03,0x5d,0x73,0x3a,0x77,0x84,0x8d,0x4e,0x49,0xd2,
    0xfb,0x91,0x6a,0xcc,0x8a,0x35,0x02,0x55,0x7a,0x34,0x96,0x3d,0xd3,0x41,0x85,0xf2,
    0xb1,0x75,0xc4,0xb5,0xbb,0xb3,0x1b,0xd5,0x07,0x05,0x17,0x0b,0x7b,0xd7,0xdf,0xea,
    0xe3,0x57,0xc0,0x95,0x9c,0x6e,0x14,0xae,0xb9,0x6b,0xc1,0x81,0x87,0x74,0xd8,0xe2,
    0xec,0x52,0xbc,0xe9,0xe1,0xdb,0x0c,0xf7,0xaf,0x5a,0x9a,0xc7,0xfa,0xf6,0xee,0xfe };

static inline int hash8(const uint8_t *s)        /* canonical hash of the 8-mer s[0..8) (GIXmake.c:530-537) */
{ int f0 = (s[0]<<6)|(s[1]<<4)|(s[2]<<2)|s[3];
  int f1 = (s[4]<<6)|(s[5]<<4)|(s[6]<<2)|s[7];
  int r0 = ((3-s[7])<<6)|((3-s[6])<<4)|((3-s[5])<<2)|(3-s[4]);   /* revcomp first 4-mer */
  int r1 = ((3-s[3])<<6)|((3-s[2])<<4)|((3-s[1])<<2)|(3-s[0]);
  int mn = (TMap[f0]<<8) | TMap[f1];
  int mc = (TMap[r0]<<8) | TMap[r1];
  return (mn < mc ? mn : mc);
}

/* Sampled syncmer start positions of one contig (bases 0..3, one per byte), by the running
   min4/pos4 automaton exactly as scan_thread walks it (GIXmake.c:516-567).  Returns count. */

int64_t orc_syncmers(const uint8_t *seq, int64_t len, int64_t *out /* >= len entries or NULL */)
{ int64_t n = 0, i, j, pos4;
  int     mzr[4], min4;

  if (len < 12) return 0;
  min4 = 0x10000; pos4 = 0;
  for (i = 0; i < 4; i++)
    { int mz = mzr[i] = hash8(seq+i);
      if (mz < min4) { min4 = mz; pos4 = i; }
    }
  for (i = 4; i <= len-8; i++)
    { int mz = hash8(seq+i);
      mzr[i&3] = mz;
      if (mz < min4)
        { min4 = mz; pos4 = i; }
      else if (pos4 == i-4)
        { min4 = mzr[(++pos4)&3];
          for (j = pos4+1; j <= i; j++)
            if (mzr[j&3] < min4)
              { min4 = mzr[j&3]; pos4 = j; }
        }
      else if (mz > min4)
        continue;
      if (out) out[n] = i-4;
      n += 1;
    }
  return n;
}

static int KCMP(const void *l, const void *r)
/* by 80-bit k-mer, then (strand|contig rank, post): the reference leaves the order of equal
   k-mers to its thread schedule (MSDsort.c, unstable); the device table fixes it by value */
{ const rec128 *a = *(const rec128 * const *) l, *b = *(const rec128 * const *) r;
  if (a->hi != b->hi) return a->hi < b->hi ? -1 : 1;
  if (a->lo != b->lo) return a->lo < b->lo ? -1 : 1;
  return a < b ? -1 : (a > b);
}

/* Build the sorted k-mer table of a genome.  seq[c] = contig c, one base per byte; crank[c] =
   rank of contig c in the length-sorted permutation (GIXmake.c:1950-1963).  Output records in
   the device layout (common.cuh), pstart[2^24+1] lower-bound prefix index.  *tab is malloc'd. */

int64_t orc_gix_build(int ncontig, const uint8_t **seq, const int64_t *clen, const int *crank,
                      rec128 **tab, uint32_t *pstart)
{ int64_t cap = 0, n = 0, c, i, q;
  for (c = 0; c < ncontig; c++) cap += 2*(clen[c] > 0 ? clen[c] : 0);
  rec128 *raw = (rec128 *) malloc(sizeof(rec128)*(cap+1));
  for (c = 0; c < ncontig; c++)
    { int64_t L = clen[c];
      if (L < 12) continue;
      int64_t *pos = (int64_t *) malloc(sizeof(int64_t)*L);
      int64_t  m = orc_syncmers(seq[c],L,pos);
      for (q = 0; q < m; q++)
        { int64_t j = pos[q];
          if (j <= L-KMER)                                     /* GIXmake.c:571-578, 944-953 */
            { uint64_t hi = 0, lo = 0;
              for (i = 0; i < 32; i++) hi = (hi<<2) | seq[c][j+i];
              for (i = 32; i < 40; i++) lo = (lo<<2) | seq[c][j+i];
              raw[n].hi = hi;
              raw[n].lo = (lo<<48) | ((uint64_t) crank[c] << 32) | (uint32_t) j;
              n += 1;
            }
          if (j >= KMER-12)                                    /* GIXmake.c:579-586, 929-942 */
            { uint64_t hi = 0, lo = 0;
              int64_t e = j+11;                                /* k-mer base i = comp(seq[e-i]) */
              for (i = 0; i < 32; i++) hi = (hi<<2) | (3-seq[c][e-i]);
              for (i = 32; i < 40; i++) lo = (lo<<2) | (3-seq[c][e-i]);
              raw[n].hi = hi;
              raw[n].lo = (lo<<48) | ((uint64_t) (crank[c] | 0x8000) << 32) | (uint32_t) (j+12);
              n += 1;
            }
        }
      free(pos);
    }
  const rec128 **ptr = (const rec128 **) malloc(sizeof(rec128 *)*(n+1));
  for (i = 0; i < n; i++) ptr[i] = raw+i;
  qsort(ptr,n,sizeof(rec128 *),KCMP);
  rec128 *srt = (rec128 *) malloc(sizeof(rec128)*(n+1));
  for (i = 0; i < n; i++) srt[i] = *ptr[i];
  free(ptr); free(raw);
  if (pstart != NULL)
    { int64_t x = 0;
      for (i = 0; i <= n; i++)
        { int64_t p = (i == n) ? (1ll<<24) : (int64_t) (srt[i].hi >> 40);
          while (x <= p) pstart[x++] = (uint32_t) i;
        }
    }
  *tab = srt;
  return n;
}

void orc_free(void *p) { free(p); }

/***********************************************************************************************
 *  B.  Adaptamer merge: new_merge_thread (FastGA.c:610-1025) restated on 128-bit records.
 *      The LCP byte of a .ktab entry is the true LCP in bases with its predecessor, 40 for a
 *      duplicate (MSDsort.c:121-127, GIXmake.c:1249-1254); here it is recomputed on the fly.
 **********************************************************************************************/

static inline int klcp(const rec128 *a, const rec128 *b)
{ uint64_t x = a->hi ^ b->hi;
  if (x) return __builtin_clzll(x) >> 1;
  uint32_t y = (uint32_t) ((a->lo ^ b->lo) >> 48);
  if (y) return 32 + ((__builtin_clz(y) - 16) >> 1);
  return 40;
}

static inline int kbase(const rec128 *a, int p)     /* base p (0..39) of the k-mer */
{ if (p < 32) return (int) (a->hi >> (62-2*p)) & 3;
  return (int) (a->lo >> (62-2*(p-32))) & 3;
}

typedef struct { uint8_t plen; uint8_t comp; uint16_t icont, jcont; uint32_t ipost, jpost; } orc_seed;

/* Walks T1 and the per-panel slice of T2 with the reference's (plen, vlcp[], rend, eorun) state
   machine.  Emits (plen, T1 entry, T2 entry) for forward T1 entries whose block is < freq.
   out may be NULL (count only).  Returns the number of seeds; *sumlen gets the sum of plen.
   orc_merge_counters() reports how often the last call took each branch of the walk (MB_*). */

enum { MB_PANEL, MB_NLCP_GT, MB_NLCP_EQ_EORUN, MB_NLCP_EQ, MB_NLCP_LT, MB_REND_SKIP, MB_NLCP_LT_EORUN,
       MB_EXT_LB, MB_EXT_GT, MB_EXT_FULL, MB_NCOUNT };
static int64_t merge_branch[MB_NCOUNT];

void orc_merge_counters(int64_t *out)
{ int k;
  for (k = 0; k < MB_NCOUNT; k++) out[k] = merge_branch[k];
}

int64_t orc_merge(const rec128 *T1, int64_t n1, const rec128 *T2, int64_t n2,
                  const uint32_t *pstart2, int freq, orc_seed *out, int64_t *sumlen)
{ int64_t nh = 0, ts = 0, i;
  int64_t cpre = -1;
  int64_t cbeg = 0, cend = 0;          /* current T2 panel [cbeg,cend) */
  int     plen = 12, eorun = 0;
  int64_t vlcp[KMER+1], rend = 0, low = 0, hgh = 0, top = 0;
  (void) n2;
  memset(merge_branch,0,sizeof(merge_branch));

#define LB(x) ((x) >= cend ? 11 : klcp(T2+(x)-1,T2+(x)))      /* ctop[LBYTE] = 11 sentinel (:719) */

  for (i = 0; i < n1; i++)
    { const rec128 *e1 = T1+i;
      int64_t pre = (int64_t) (e1->hi >> 40);
      if (pre != cpre)                                  /* new prefix panel (:686-744) */
        { cpre = pre;
          cbeg = pstart2[pre]; cend = pstart2[pre+1];
          if (cbeg == cend)                             /* empty cache: skip the T1 panel */
            { while (i+1 < n1 && (int64_t) (T1[i+1].hi >> 40) == pre) i += 1;
              cpre = -1;
              continue;
            }
          merge_branch[MB_PANEL] += 1;
          plen = 12;
          vlcp[plen] = rend = cbeg;
          eorun = 0;
        }
      else
        { int nlcp = klcp(T1+i-1,e1);                   /* suf1[LBYTE] (:752) */
          if (nlcp > plen)
            { merge_branch[MB_NLCP_GT] += 1;
              goto pairs;
            }
          else if (nlcp == plen)
            { merge_branch[eorun ? MB_NLCP_EQ_EORUN : MB_NLCP_EQ] += 1;
              if (eorun) goto pairs;
            }
          else
            { int64_t r0;
              merge_branch[MB_NLCP_LT] += 1;
              if (!eorun) rend += 1;
              r0 = rend;
              while (LB(rend) > nlcp) rend += 1;
              if (rend > r0) merge_branch[MB_REND_SKIP] += 1;
              plen = LB(rend);
              if (plen < nlcp)
                { merge_branch[MB_NLCP_LT_EORUN] += 1;
                  eorun = 1; plen = nlcp; goto range;
                }
              eorun = 0;
            }
        }

      while (plen < KMER)                               /* extend the match (:775-792) */
        { int c = kbase(e1,plen), d;
          for (d = kbase(T2+rend,plen); d < c; d = kbase(T2+rend,plen))
            { rend += 1;
              if (LB(rend) < plen)
                { merge_branch[MB_EXT_LB] += 1;
                  eorun = 1; goto range;
                }
            }
          if (d > c)
            { merge_branch[MB_EXT_GT] += 1;
              goto range;
            }
          plen += 1;
          vlcp[plen] = rend;
        }
      merge_branch[MB_EXT_FULL] += 1;
      do rend += 1; while (LB(rend) >= KMER);
      eorun = 1;

    range:                                              /* full T2 range (:796-807) */
      low = vlcp[plen];
      hgh = rend;
      top = low + freq;
      if (!eorun)
        { do
            { hgh += 1;
              if (hgh > top) break;
            }
          while (LB(hgh) >= plen);
        }

    pairs:
      if (hgh >= top) continue;                         /* :817 */
      if ((e1->lo >> 47) & 1) continue;                 /* reverse-strand T1 entry (:921-928) */
      { int64_t p;
        for (p = low; p < hgh; p++)
          { if (out)
              { orc_seed *s = out+nh;
                s->plen  = (uint8_t) plen;
                s->comp  = (uint8_t) ((T2[p].lo >> 47) & 1);
                s->icont = (uint16_t) ((e1->lo >> 32) & 0x7fff);
                s->jcont = (uint16_t) ((T2[p].lo >> 32) & 0x7fff);
                s->ipost = (uint32_t) e1->lo;
                s->jpost = (uint32_t) T2[p].lo;
              }
            nh += 1;
            ts += plen;
          }
      }
    }
#undef LB
  if (sumlen) *sumlen = ts;
  return nh;
}

/*  SELF mode (FastGA A): new_self_merge_thread (FastGA.c:1616-1909).  T2 is T1.  EVERY entry,
    either strand, is an i: plen = its longest prefix shared with another entry of its 12-base
    panel (max of the LCPs with its two neighbours), block = the run of entries sharing those plen
    bases, entry included; if the block has < freq members, one pair (i, p) for every OTHER member
    p, strand C iff the signs differ (:1801-1860).  Both orders of a pair come out; the reference
    reports half the count (:1907).  Declarative restatement of the (plen, vlcp[], rend, eorun)
    machine at :1707-1790.  */

int64_t orc_self_merge(const rec128 *T, int64_t n, const uint32_t *pstart, int freq,
                       orc_seed *out, int64_t *sumlen)
{ int64_t nh = 0, ts = 0, i;
  for (i = 0; i < n; i++)
    { int64_t pre  = (int64_t) (T[i].hi >> 40);
      int64_t cbeg = pstart[pre], cend = pstart[pre+1];
      int lp = (i > cbeg)   ? klcp(T+i-1,T+i) : 11;
      int ls = (i+1 < cend) ? klcp(T+i,T+i+1) : 11;
      int plen = lp > ls ? lp : ls;
      int64_t lo = i, hi = i+1, p;
      if (plen < 12) continue;                              /* alone in its panel: block = itself */
      while (lo > cbeg && klcp(T+lo-1,T+lo) >= plen) lo -= 1;
      while (hi < cend && hi - lo < freq && klcp(T+hi-1,T+hi) >= plen) hi += 1;
      if (hi - lo >= freq) continue;
      for (p = lo; p < hi; p++)
        { if (p == i) continue;
          if (out)
            { orc_seed *s = out+nh;
              s->plen  = (uint8_t) plen;
              s->comp  = (uint8_t) ((((T[i].lo >> 47) ^ (T[p].lo >> 47)) & 1));
              s->icont = (uint16_t) ((T[i].lo >> 32) & 0x7fff);
              s->jcont = (uint16_t) ((T[p].lo >> 32) & 0x7fff);
              s->ipost = (uint32_t) T[i].lo;
              s->jpost = (uint32_t) T[p].lo;
            }
          nh += 1;
          ts += plen;
        }
    }
  if (sumlen) *sumlen = ts;
  return nh;
}

/***********************************************************************************************
 *  C.  Seed records (reimport_thread, FastGA.c:2703-2721) and their order (RSDsort.c: key read
 *      from the last byte backwards = jcont, band, anti, diag&63, lcp), here with strand and
 *      icont on top so one sort covers every (strand, A-contig) panel.
 **********************************************************************************************/

typedef struct { int anti_bits, band_bits, jc_bits, ic_bits; int64_t amxpos, bmxpos; } orc_layout;

static inline void put_bits(rec128 *r, int pos, uint64_t v)
{ if (pos < 64)
    { r->lo |= v << pos;
      if (pos > 0) r->hi |= v >> (64-pos);
    }
  else
    r->hi |= v << (pos-64);
}

static inline uint64_t get_bits(const rec128 *r, int pos, int n)
{ uint64_t v;
  if (n == 0) return 0;
  if (pos >= 64) v = r->hi >> (pos-64);
  else if (pos == 0) v = r->lo;
  else v = (r->lo >> pos) | (r->hi << (64-pos));
  return n >= 64 ? v : (v & ((1ull<<n)-1));
}

static int SCMP(const void *l, const void *r)
{ const rec128 *a = (const rec128 *) l, *b = (const rec128 *) r;
  if (a->hi != b->hi) return a->hi < b->hi ? -1 : 1;
  if (a->lo != b->lo) return a->lo < b->lo ? -1 : 1;
  return 0;
}

void orc_seed_records(const orc_seed *s, int64_t n, const orc_layout *L, rec128 *out, int do_sort)
{ int64_t i;
  for (i = 0; i < n; i++)
    { int64_t ip = s[i].ipost, jp = s[i].jpost, diag, anti;
      if (s[i].comp)
        { diag = (L->amxpos + L->bmxpos) - (ip+jp); anti = L->amxpos - (ip-jp); }
      else
        { diag = L->bmxpos + (ip-jp); anti = ip+jp; }
      rec128 r = {0,0};
      int pos = 0;
      put_bits(&r,pos,s[i].plen);          pos += 6;
      put_bits(&r,pos,(uint64_t) (diag&63)); pos += 6;
      put_bits(&r,pos,(uint64_t) anti);    pos += L->anti_bits;
      put_bits(&r,pos,(uint64_t) (diag>>6)); pos += L->band_bits;
      put_bits(&r,pos,s[i].jcont);         pos += L->jc_bits;
      put_bits(&r,pos,s[i].icont);         pos += L->ic_bits;
      put_bits(&r,pos,s[i].comp);
      out[i] = r;
    }
  if (do_sort)
    qsort(out,n,sizeof(rec128),SCMP);
}

/***********************************************************************************************
 *  D.  Wave extension: forward_wave (align.c:352-874), reverse_wave (:878-1418) and
 *      Local_Alignment (:1423-1576), folded into one direction-normalised wave.
 *
 *  Normalisation: s = +1 forward, -1 reverse; kk = s*k, xn = s*x, values W = s*V.  In these
 *  coordinates the reverse wave IS the forward wave (predecessor choice, tie order of the
 *  running maxima, band growth / clip / trim), except for: the wave-0 start (floor((mida+k)/2)
 *  in ORIGINAL coordinates), the root pebble (forward: mark = trace point at or below x,
 *  reverse: mark = x itself, align.c:441-453 vs :969-979), the "fresh" value given to new band
 *  edges (-1 vs INT32_MAX) and the trace read-out.
 **********************************************************************************************/

#define TRIM_LEN    15
#define DUB_TRIM    45
#define PATH_LEN    60
#define PATH_TOP    0x1000000000000000ull
#define PATH_INT    0x0fffffffffffffffull
#define PATH_WIN    0x1fffffffffffffffull      /* M = popcount(T & PATH_WIN), see align.c:677-702 */
#define TRIM_MASK   0x7fff
#define TRIM_MLAG   250
#define WAVE_LAG    70

typedef struct { int ptr, diag, diff, mark; } Peb;

typedef struct
  { int      tspace, path_ave;
    int16_t *score, *table;              /* 32768 entries each (align.c:207-268) */
  } orc_spec;

static const double Bias_Factor[10] = { .690, .690, .690, .690, .780, .850, .900, .933, .966, 1.000 };

static void set_table(int bit, int prefix, int score, int max, int mscore, int dscore,
                      int16_t *table, int16_t *sc)
{ if (bit >= TRIM_LEN)
    { table[prefix] = (int16_t) (score-max);
      sc[prefix]    = (int16_t) score;
    }
  else
    { if (score > max) max = score;
      set_table(bit+1,(prefix<<1),  score-dscore,max,mscore,dscore,table,sc);
      set_table(bit+1,(prefix<<1)|1,score+mscore,max,mscore,dscore,table,sc);
    }
}

/* New_Align_Spec (align.c:222-268): float/double set-up -> two int16 tables + ave_path.
   tables: 2 x 32768 int16, score first then table (same as the reference allocation). */

int orc_align_spec(double ave_corr, const float *freq, int16_t *tables, int *ave_path)
{ double match;
  int    bias, mscore, dscore;
  match = freq[0] + freq[3];
  if ((match <= 0.) == (match > 0.)) match = .5;
  if (match > .5) match = 1.-match;
  bias = (int) ((match+.025)*20.-1.);
  if (match < .2) bias = 3;
  *ave_path = (int) (PATH_LEN * (1. - Bias_Factor[bias] * (1. - ave_corr)));
  mscore    = (int) (1000 * Bias_Factor[bias] * (1. - ave_corr));
  dscore    = 1000 - mscore;
  set_table(0,0,0,0,mscore,dscore,tables+(TRIM_MASK+1),tables);
  return 0;
}

/*  What one wave pass went through (orc_search_calls): the regimes a device wave routine branches on.
    Coordinates are the pass's own (direction-normalised); `call` is the Local_Alignment call's number.  */
typedef struct
  { int call, s;
    int waves;                   /* waves after wave 0 */
    int maxband;                 /* widest band a wave ran over (hghk-lowk+1 after the band grew) */
    int narrowspan;              /* most A bases the best point advanced over consecutive waves of <= 17 diagonals */
    int maxsnake;                /* longest slide of one diagonal in one wave after wave 0 */
    int aend, bend;              /* a slide met the end of A (ca == 4) / of B (cb == 4) */
    int stall;                   /* a wave after wave 0 did not raise besta: never, see wave() */
    int endempty;                /* a wave stopped by a contig end left no diagonal after the end clip and trim */
    int aspan;                   /* A bases from the start point to the trim point */
    int da0, da1, db0, db1;      /* the start point's distance to A's start, A's end, B's start, B's end */
    int maxhop;                  /* largest cell-index gap between consecutive pebbles of the read-out path */
  } orc_pass;

/*  Every Local_Alignment call of orc_search_calls in discovery order: its arguments (original contig
    numbers), whether it produced a record, its path (trace bytes at toff in tpool), its passes.  */
typedef struct
  { int comp, ctg1, ctg2, low, hgh, anti, lbord, hbord, rec;
    int abpos, bbpos, aepos, bepos, diffs, tlen, pass0, npass, pad;
    int64_t toff;
  } orc_call;

typedef struct
  { orc_call *call; int64_t ncall, maxcall;
    uint8_t  *tpool; int64_t tlen, tmax;
    orc_pass *pass; int64_t npass, maxpass;
  } orc_calllog;

static orc_pass *pass_new(orc_calllog *g)
{ if (g == NULL) return NULL;
  if (g->npass >= g->maxpass)
    { g->maxpass = g->maxpass*2 + 256;
      g->pass = (orc_pass *) realloc(g->pass,sizeof(orc_pass)*g->maxpass);
    }
  orc_pass *p = g->pass + g->npass++;
  memset(p,0,sizeof(orc_pass));
  p->call = (int) g->ncall;
  return p;
}

typedef struct
  { const char *aseq, *bseq;     /* one base per byte, sentinel 4 at [-1] and [len] */
    int   alen, blen;
    int   W;                     /* state capacity (power of two), circular on kk   */
    int      *V, *HA, *NA;
    uint64_t *T;
    Peb  *cells;
    int   cmax, avail;
    orc_calllog *log;            /* NULL, or where orc_local_alignment records its passes */
  } orc_work;

static inline int a_at(const orc_work *w, int s, int xn)
{ int i = (s > 0) ? xn : -xn-1;
  return (i < 0 || i >= w->alen) ? 4 : w->aseq[i];
}
static inline int b_at(const orc_work *w, int s, int yn)
{ int i = (s > 0) ? yn : -yn-1;
  return (i < 0 || i >= w->blen) ? 4 : w->bseq[i];
}

static void grow_state(orc_work *w, int lowk, int hghk)   /* keeps [lowk-1,hghk+1] valid */
{ int need = (hghk - lowk) + 9, nW = w->W, k;
  if (need <= w->W) return;
  while (nW < need) nW *= 2;
  int      *V  = (int *) malloc(sizeof(int)*nW), *HA = (int *) malloc(sizeof(int)*nW);
  int      *NA = (int *) malloc(sizeof(int)*nW);
  uint64_t *T  = (uint64_t *) malloc(sizeof(uint64_t)*nW);
  for (k = lowk-1; k <= hghk+1; k++)
    { int o = k & (w->W-1), n = k & (nW-1);
      V[n] = w->V[o]; HA[n] = w->HA[o]; NA[n] = w->NA[o]; T[n] = w->T[o];
    }
  free(w->V); free(w->HA); free(w->NA); free(w->T);
  w->V = V; w->HA = HA; w->NA = NA; w->T = T; w->W = nW;
}

static inline int new_cell(orc_work *w, int ptr, int diag, int diff, int mark)
{ if (w->avail >= w->cmax)
    { w->cmax  = (int) (w->avail*1.2) + 10000;
      w->cells = (Peb *) realloc(w->cells,sizeof(Peb)*w->cmax);
    }
  Peb *p = w->cells + w->avail;
  p->ptr = ptr; p->diag = diag; p->diff = diff; p->mark = mark;
  return w->avail++;
}

typedef struct
  { int endx, endy;       /* trim point, ORIGINAL coordinates */
    int diffs;
    int trimha;
    int root_diag;        /* diagonal on which the winning path started (forward *mind) */
  } wave_out;

#define IX(k) ((k) & Wm)

static void wave(orc_work *w, const orc_spec *spec, int s, int low, int hgh, int mida,
                 int minp, int maxp, int aoff, wave_out *out, orc_pass *st)
{ int tspace = spec->tspace, PATH_AVE = spec->path_ave;
  const int16_t *SCORE = spec->score, *TABLE = spec->table;
  int FRESH = (s > 0) ? -1 : -INT32_MAX;
  int lowk, hghk, minpn, maxpn, dif;
  int besta, bestx, lasta, trima, trimx, trimd, trimha;
  int more, aclip, bclip, Wm, kk;
  int nx0 = 0, nrun = 0;                               /* pass statistics: start of the current narrow stretch */

  if (s > 0) { lowk = low;  hghk = hgh;  minpn = minp;  maxpn = maxp; }
  else       { lowk = -hgh; hghk = -low; minpn = -maxp; maxpn = -minp; }

  grow_state(w,lowk,hghk);
  Wm = w->W-1;
  w->avail = 0;
  dif  = 0;
  more = 1;
  aclip = INT32_MAX; bclip = -INT32_MAX;

  besta = trima = lasta = s*mida;
  bestx = trimx = s*((mida+hgh)>>1);
  trimd = 0; trimha = 0;
  if (st != NULL)
    { int xm = (mida + ((low+hgh)>>1))>>1, ym = mida - xm;
      st->s = s;
      st->da0 = xm; st->da1 = w->alen - xm; st->db0 = ym; st->db1 = w->blen - ym;
      st->maxband = hghk - lowk + 1;
    }

  for (kk = hghk; kk >= lowk; kk--)                    /* wave 0 (align.c:426-507 / :956-1036) */
    { int k = s*kk, x = (mida+k)>>1, xn, na, nan, ha, c;
      if (s > 0)
        { na  = ((x+(tspace-aoff))/tspace-1)*tspace+aoff;
          ha  = new_cell(w,-1,k,0,na);
          nan = na + tspace;
        }
      else
        { na  = ((x+(tspace-aoff)-1)/tspace-1)*tspace+aoff;
          ha  = new_cell(w,-1,k,0,x);
          nan = -na;
        }
      xn = s*x;
      while (1)
        { int cb = b_at(w,s,xn-kk), ca;
          if (cb == 4)
            { more = 0;
              if (bclip < kk) bclip = kk;
              if (st != NULL) st->bend = 1;
              break;
            }
          ca = a_at(w,s,xn);
          if (cb != ca)
            { if (ca == 4) { more = 0; aclip = kk; if (st != NULL) st->aend = 1; }
              break;
            }
          xn += 1;
        }
      c = 2*xn - kk;
      while (xn >= nan)
        { ha = new_cell(w,ha,k,0,s*nan);
          nan += tspace;
        }
      if (c > besta)
        { besta = trima = lasta = c;
          bestx = trimx = xn;
          trimha = ha;
        }
      w->V[IX(kk)] = c; w->T[IX(kk)] = PATH_INT; w->HA[IX(kk)] = ha; w->NA[IX(kk)] = nan;
    }

  if (more == 0)
    { if (b_at(w,s,besta-bestx) != 4 && a_at(w,s,bestx) != 4) more = 1;
      if (hghk >= aclip) hghk = aclip-1;
      if (lowk <= bclip) lowk = bclip+1;
      aclip = INT32_MAX; bclip = -INT32_MAX;
    }

  while (more && lasta >= besta - TRIM_MLAG)           /* align.c:546-800 / :1077-1330 */
    { int am, ac, ap, ua, n, besta0 = besta;
      uint64_t t;

      grow_state(w,lowk-1,hghk+1);
      Wm = w->W-1;
      lowk -= 1; hghk += 1;

      if (lowk >= minpn)
        { w->NA[IX(lowk)] = w->NA[IX(lowk+1)]; w->V[IX(lowk)] = FRESH; }
      else
        lowk += 1;
      if (hghk <= maxpn)
        { w->NA[IX(hghk)] = w->NA[IX(hghk-1)]; w->V[IX(hghk)] = FRESH; }
      else
        hghk -= 1;
      dif += 1;
      if (st != NULL)
        { st->waves += 1;
          if (hghk - lowk + 1 > st->maxband) st->maxband = hghk - lowk + 1;
          if (hghk - lowk + 1 > 17)
            nrun = 0;
          else
            { if (!nrun) { nrun = 1; nx0 = bestx; }
              if (bestx - nx0 > st->narrowspan) st->narrowspan = bestx - nx0;
            }
        }

      w->V[IX(hghk+1)] = w->V[IX(lowk-1)] = FRESH;
      ac = FRESH;
      am = w->V[IX(hghk)];
      t  = PATH_INT;
      ua = -1;
      for (kk = hghk; kk >= lowk; kk--)
        { int xn, x0, c, ha, k = s*kk;
          uint64_t b;

          ap = ac; ac = am; am = w->V[IX(kk-1)];
          if (ac < am)
            { if (am < ap) { c = ap+1; b = t; ha = ua; }
              else         { c = am+1; b = w->T[IX(kk-1)]; ha = w->HA[IX(kk-1)]; }
            }
          else
            { if (ac < ap) { c = ap+1; b = t; ha = ua; }
              else         { c = ac+2; b = w->T[IX(kk)]; ha = w->HA[IX(kk)]; }
            }
          b <<= 1;
          xn = x0 = (c+kk)>>1;
          while (1)
            { int cb = b_at(w,s,xn-kk), ca;
              if (cb == 4)
                { more = 0;
                  if (bclip < kk) bclip = kk;
                  if (st != NULL) st->bend = 1;
                  break;
                }
              ca = a_at(w,s,xn);
              if (cb != ca)
                { if (ca == 4) { more = 0; aclip = kk; if (st != NULL) st->aend = 1; }
                  break;
                }
              xn += 1;
              b = (b << 1) | 1;
            }
          if (st != NULL && xn - x0 > st->maxsnake) st->maxsnake = xn - x0;
          c = 2*xn - kk;

          while (xn >= w->NA[IX(kk)])
            { if (s*w->cells[ha].mark < w->NA[IX(kk)])
                ha = new_cell(w,ha,k,dif,s*w->NA[IX(kk)]);
              w->NA[IX(kk)] += tspace;
            }

          if (c > besta)
            { besta = c; bestx = xn;
              if (__builtin_popcountll(b & PATH_WIN) >= PATH_AVE)
                { lasta = c;
                  if (TABLE[b & TRIM_MASK] >= 0)
                    if (TABLE[(b >> TRIM_LEN) & TRIM_MASK] + SCORE[b & TRIM_MASK] >= 0)
                      { trima = c; trimx = xn; trimd = dif; trimha = ha; }
                }
            }

          t  = w->T[IX(kk)];
          ua = w->HA[IX(kk)];
          w->V[IX(kk)] = c; w->T[IX(kk)] = b; w->HA[IX(kk)] = ha;
        }

      /* besta cannot stall: the diagonal holding it gains at least 2 each wave while it is in the band, the
         WAVE_LAG trim never drops it, and an end clip drops it only when it slid into that end itself (a
         diagonal at or above aclip with as large a value lies as far along A; at or below bclip, along B),
         which leaves more == 0.  The device's "no advance" bail-out is reached the other way: the wave
         that meets an end leaves no diagonal within WAVE_LAG once the clipped ones are gone (endempty). */
      if (st != NULL && besta == besta0) st->stall = 1;
      if (more == 0)
        { if (b_at(w,s,besta-bestx) != 4 && a_at(w,s,bestx) != 4) more = 1;
          if (hghk >= aclip) hghk = aclip-1;
          if (lowk <= bclip) lowk = bclip+1;
          aclip = INT32_MAX; bclip = -INT32_MAX;
        }

      n = besta - WAVE_LAG;
      while (hghk >= lowk)
        if (w->V[IX(hghk)] < n)
          hghk -= 1;
        else
          { while (w->V[IX(lowk)] < n) lowk += 1;
            break;
          }
      if (st != NULL && more == 0 && hghk < lowk) st->endempty = 1;
    }

  out->endx   = s*trimx;
  out->endy   = s*(trima - trimx);
  out->diffs  = trimd;
  out->trimha = trimha;
  if (st != NULL)
    { int h;
      st->aspan = trimx - s*((mida+hgh)>>1);
      for (h = trimha; w->cells[h].ptr >= 0; h = w->cells[h].ptr)
        if (h - w->cells[h].ptr > st->maxhop) st->maxhop = h - w->cells[h].ptr;
    }
  { int h = trimha;
    while (w->cells[h].ptr >= 0) h = w->cells[h].ptr;
    out->root_diag = w->cells[h].diag;
  }
}

typedef struct
  { int abpos, bbpos, aepos, bepos, diffs, tlen;
    uint8_t *trace;              /* tlen bytes (Compress_TraceTo8 without check, align.c:3892) */
    int      tmax;
  } orc_path;

static void tr_reserve(orc_path *p, int n)
{ if (n > p->tmax)
    { p->tmax  = n*2 + 64;
      p->trace = (uint8_t *) realloc(p->trace,p->tmax);
    }
}

/* forward read-out (align.c:805-870): pairs (diff delta, B advance) root -> tip, appended */

static void fwd_trace(orc_work *w, const wave_out *r, int mida, orc_path *p)
{ int n = 0, h, i, k, a, b, d, e, trimx = r->endx, trimy = r->endy, trimd = r->diffs;
  for (h = r->trimha; h >= 0; h = w->cells[h].ptr) n += 1;
  int *chain = (int *) malloc(sizeof(int)*n);
  for (h = r->trimha, i = n-1; h >= 0; h = w->cells[h].ptr) chain[i--] = h;
  k = w->cells[chain[0]].diag;
  b = (mida-k)>>1;
  e = 0;
  tr_reserve(p,p->tlen+2*n+2);
  for (i = 1; i < n; i++)
    { h = chain[i];
      k = w->cells[h].diag;
      a = w->cells[h].mark - k;
      d = w->cells[h].diff;
      p->trace[p->tlen++] = (uint8_t) (d-e);
      p->trace[p->tlen++] = (uint8_t) (a-b);
      b = a; e = d;
    }
  if (b+k != trimx)
    { p->trace[p->tlen++] = (uint8_t) (trimd-e);
      p->trace[p->tlen++] = (uint8_t) (trimy-b);
    }
  else if (b != trimy && p->tlen >= 2)     /* with no pair the reference's write lands in scratch */
    { p->trace[p->tlen-1] = (uint8_t) (p->trace[p->tlen-1] + (trimy-b));
      p->trace[p->tlen-2] = (uint8_t) (p->trace[p->tlen-2] + (trimd-e));
    }
  free(chain);
  p->aepos = trimx; p->bepos = trimy; p->diffs = trimd;
}

/* reverse read-out (align.c:1334-1414): pairs are PREPENDED to whatever trace p already holds */

static void rev_trace(orc_work *w, const wave_out *r, int tspace, int aoff, orc_path *p)
{ int n = 0, h, i, k, a, b, d, e, trimx = r->endx, trimy = r->endy, trimd = r->diffs;
  for (h = r->trimha; h >= 0; h = w->cells[h].ptr) n += 1;
  int *chain = (int *) malloc(sizeof(int)*n);
  for (h = r->trimha, i = n-1; h >= 0; h = w->cells[h].ptr) chain[i--] = h;
  uint8_t *pre = (uint8_t *) malloc(2*n+4);        /* generated order; final = reversed pairs */
  int np = 0, ci = 0, live = 1;

  k = w->cells[chain[0]].diag;
  b = w->cells[chain[0]].mark - k;
  e = 0; d = 0;
  if ((b+k)%tspace != aoff)
    { ci = 1;
      if (ci >= n)
        { live = 0; a = trimy; d = trimd; }
      else
        { h = chain[ci];
          k = w->cells[h].diag;
          a = w->cells[h].mark - k;
          d = w->cells[h].diff;
        }
      if (p->tlen == 0)
        { pre[np++] = (uint8_t) (d-e); pre[np++] = (uint8_t) (b-a); }
      else
        { p->trace[1] = (uint8_t) (p->trace[1] + (b-a));
          p->trace[0] = (uint8_t) (p->trace[0] + (d-e));
        }
      b = a; e = d;
    }
  if (live)
    { for (ci = ci+1; ci < n; ci++)
        { h = chain[ci];
          k = w->cells[h].diag;
          a = w->cells[h].mark - k;
          d = w->cells[h].diff;
          pre[np++] = (uint8_t) (d-e); pre[np++] = (uint8_t) (b-a);
          b = a; e = d;
        }
      if (b+k != trimx)
        { pre[np++] = (uint8_t) (trimd-e); pre[np++] = (uint8_t) (b-trimy); }
      else if (b != trimy)
        { /* adjusts the most recently prepended pair = the first pair of the final trace;
             if nothing was prepended that is the first pair already in p (atrace[atlen]) */
          if (np >= 2)
            { pre[np-1] = (uint8_t) (pre[np-1] + (b-trimy));
              pre[np-2] = (uint8_t) (pre[np-2] + (trimd-e));
            }
          else if (p->tlen >= 2)
            { p->trace[1] = (uint8_t) (p->trace[1] + (b-trimy));
              p->trace[0] = (uint8_t) (p->trace[0] + (trimd-e));
            }
        }
    }
  tr_reserve(p,p->tlen+np+2);
  memmove(p->trace+np,p->trace,p->tlen);
  for (i = 0; i < np; i += 2)
    { p->trace[np-2-i] = pre[i];
      p->trace[np-1-i] = pre[i+1];
    }
  p->tlen += np;
  free(pre); free(chain);
  p->abpos = trimx; p->bbpos = trimy; p->diffs += trimd;
}

orc_work *orc_new_work(void)
{ orc_work *w = (orc_work *) calloc(1,sizeof(orc_work));
  w->W  = 1024;
  w->V  = (int *) malloc(sizeof(int)*w->W);  w->HA = (int *) malloc(sizeof(int)*w->W);
  w->NA = (int *) malloc(sizeof(int)*w->W);  w->T  = (uint64_t *) malloc(sizeof(uint64_t)*w->W);
  return w;
}

void orc_free_work(orc_work *w)
{ free(w->V); free(w->HA); free(w->NA); free(w->T); free(w->cells); free(w); }

/* Local_Alignment (align.c:1423-1576).  acomp != 0: aseq is the reverse complement of the
   contig (ACOMP_FLAG): trace-point offset aoff = alen % tspace, result flipped at the end. */

int orc_local_alignment(orc_work *w, const orc_spec *spec, const char *aseq, int alen,
                        const char *bseq, int blen, int acomp, int low, int hgh, int anti,
                        int lbord, int hbord, orc_path *p)
{ int minp, maxp, aoff, fshort, rshort, selfie;
  wave_out f, r;

  w->aseq = aseq; w->bseq = bseq; w->alen = alen; w->blen = blen;
  selfie = (aseq == bseq);
  while (((anti-hgh)>>1) < 0) hgh -= 1;
  if (lbord < 0) minp = (selfie && low >= 0) ? 1 : -INT32_MAX; else minp = low-lbord;
  if (hbord < 0) maxp = (selfie && hgh <= 0) ? -1 : INT32_MAX; else maxp = hgh+hbord;
  aoff = acomp ? alen % spec->tspace : 0;

  p->tlen = 0; p->diffs = 0;
  wave(w,spec,+1,low,hgh,anti,minp,maxp,aoff,&f,pass_new(w->log));
  fwd_trace(w,&f,anti,p);
  low = f.root_diag;
  fshort = ((p->aepos + p->bepos) - anti < DUB_TRIM);

  wave(w,spec,-1,low,low,anti,minp,maxp,aoff,&r,pass_new(w->log));
  rev_trace(w,&r,spec->tspace,aoff,p);
  rshort = (anti - (p->abpos + p->bbpos) < DUB_TRIM);

  if (fshort)
    { if (rshort)
        { p->aepos = p->abpos = (p->abpos+p->aepos)>>1;
          p->bepos = p->bbpos = (p->bbpos+p->bepos)>>1;
          p->tlen  = 0;
        }
      else
        { low  = p->abpos - p->bbpos;
          anti = p->abpos + p->bbpos;
          p->tlen = 0;
          wave(w,spec,+1,low,low,anti,minp,maxp,aoff,&f,pass_new(w->log));
          fwd_trace(w,&f,anti,p);
        }
    }
  else if (rshort)
    { low  = p->aepos - p->bepos;
      anti = p->aepos + p->bepos;
      p->tlen = 0; p->diffs = 0;
      wave(w,spec,-1,low,low,anti,minp,maxp,aoff,&r,pass_new(w->log));
      rev_trace(w,&r,spec->tspace,aoff,p);
    }

  if (acomp)
    { int i, j;
      i = p->abpos; p->abpos = alen - p->aepos; p->aepos = alen - i;
      i = p->bbpos; p->bbpos = blen - p->bepos; p->bepos = blen - i;
      for (i = p->tlen-2, j = 0; j < i; i -= 2, j += 2)
        { uint8_t t;
          t = p->trace[i];   p->trace[i]   = p->trace[j];   p->trace[j]   = t;
          t = p->trace[i+1]; p->trace[i+1] = p->trace[j+1]; p->trace[j+1] = t;
        }
    }
  return 0;
}

/***********************************************************************************************
 *  E.  Seed-chain detection + extension driver: align_contigs, search part
 *      (FastGA.c:2973-3403) over the sorted seed records of section C.
 *
 *  Sorted order = (strand, A-contig rank, B-contig rank, band = diag>>6, anti, diag&63, lcp).
 *  A "triple" is two adjacent 64-wide bands scanned together (b,m,e); the chain scan, the tube
 *  stepping and the alast blocking follow the reference statement by statement.
 **********************************************************************************************/

typedef struct
  { int chain_break, chain_min, align_min; double align_rate; } orc_params;

typedef struct
  { int comp, aread, bread;                 /* ORIGINAL contig numbers (Perm applied, :3007-3008) */
    int abpos, bbpos, aepos, bepos, diffs, tlen;
    int grp;                                /* index of the align_contigs call that found it */
    int64_t toff;                           /* offset of the trace bytes in the trace pool */
  } orc_ovl;

typedef struct
  { orc_ovl *ovl; int64_t novl, maxovl;
    uint8_t *tpool; int64_t tlen, tmax;
    int64_t nhit;
  } orc_result;

static void res_push(orc_result *R, const orc_ovl *o, const uint8_t *trace)
{ if (R->novl >= R->maxovl)
    { R->maxovl = R->maxovl*2 + 1024;
      R->ovl = (orc_ovl *) realloc(R->ovl,sizeof(orc_ovl)*R->maxovl);
    }
  if (R->tlen + o->tlen > R->tmax)
    { R->tmax = (R->tlen + o->tlen)*2 + 4096;
      R->tpool = (uint8_t *) realloc(R->tpool,R->tmax);
    }
  R->ovl[R->novl] = *o;
  R->ovl[R->novl].toff = R->tlen;
  memcpy(R->tpool+R->tlen,trace,o->tlen);
  R->tlen += o->tlen;
  R->novl += 1;
}

orc_result *orc_new_result(void) { return (orc_result *) calloc(1,sizeof(orc_result)); }
void orc_free_result(orc_result *R) { free(R->ovl); free(R->tpool); free(R); }
int64_t  orc_result_count(orc_result *R) { return R->novl; }
int64_t  orc_result_hits(orc_result *R) { return R->nhit; }
orc_ovl *orc_result_ovls(orc_result *R) { return R->ovl; }
uint8_t *orc_result_traces(orc_result *R) { return R->tpool; }

#define BUCK_SHIFT 6
#define BUCK_WIDTH 64
#define BUCK_ANTI  128

/*  SELF mode of align_contigs (FastGA.c:3030, :3247-3262): a contig against itself, forward
    strand, is aligned strictly above or strictly below the main diagonal and not at all across
    it.  In that last branch the reference only clears abpos/aepos, so the tube advances with the
    bepos of the previous alignment (the orc_path below persists across calls, as Path does).
    orc_set_straddle(1) advances it with 0 instead, as the CUDA path does; 0 (the default) is the
    reference.  orc_self_counters reads what the last search went through: [0] straddles (calls not
    made), [1] straddles where the previous bepos was past alow (the two advances differ), [2] calls
    with lbord >= 0, [3] calls with hbord >= 0.  */
static int g_self = 0, g_straddle_zero = 0;
static int64_t g_self_cnt[4];
void orc_set_self(int on) { g_self = on; }
void orc_set_straddle(int zero) { g_straddle_zero = zero; }
void orc_self_counters(int64_t *out) { memcpy(out,g_self_cnt,sizeof(g_self_cnt)); }

/* aseq[c], bseq[c]: contig c (ORIGINAL numbering), one base per byte with a sentinel 4 at [-1]
   and [len]; acseq[c]: reverse complement of A contig c, same framing (Complement_Seq). */

/*  The chain scan of every band-pair triple (FastGA.c:3087-3162), shared by orc_search, which
    extends each chain, and orc_chains, which only lists them.  For every scanned triple tri() is
    called first, then hit() for every chain that qualifies, in discovery order, with the values
    the scan holds at the reference's hit count (FastGA.c:3160): anti-diagonals and band-relative
    diagonals of the triple's own seeds, before any strand or offset adjustment -- the coordinates
    of the device's ChainHit -- and the number of seeds of the chain.  */
typedef struct
  { int64_t b, m, e, cdiag; uint64_t key; int isnew; } orc_triple;

typedef void (*orc_tri_fn)(void *ctx, const orc_triple *T);
typedef void (*orc_hit_fn)(void *ctx, const orc_triple *T, int64_t alow, int64_t ahgh, int dgmin, int dgmax,
                           int64_t nseed);

static void chain_scan(const rec128 *seeds, int64_t n, const orc_layout *L, int chain_break, int chain_min,
                       orc_tri_fn tri, orc_hit_fn hit, void *ctx)
{ int p_anti = 12, p_band = p_anti + L->anti_bits, p_jc = p_band + L->band_bits;
  int64_t g0 = 0;

#define ANTI(i) ((int64_t) get_bits(seeds+(i),p_anti,L->anti_bits))
#define BAND(i) ((int64_t) get_bits(seeds+(i),p_band,L->band_bits))
#define GRP(i)  (get_bits(seeds+(i),p_jc,L->jc_bits + L->ic_bits + 1))

  while (g0 < n)
    { int64_t g1 = g0;
      uint64_t gk = GRP(g0);
      while (g1 < n && GRP(g1) == gk) g1 += 1;
      { orc_triple T;
        int64_t b, m, e, cdiag;
        int     isnew, aux;

        b = e = g0;
        cdiag = BAND(e);
        while (e < g1 && BAND(e) == cdiag) e += 1;
        isnew = 1;
        while (1)
          { m = e; aux = 0;
            while (e < g1 && BAND(e) == cdiag+1) { e += 1; aux = 1; }

            if (isnew || aux)
              { int     go, lcp, wch, mix, cov, dgmin, dgmax, dg;
                int64_t ahgh, alow, anti, ipost, apost, s, t, nseed;

                T.b = b; T.m = m; T.e = e; T.cdiag = cdiag; T.key = gk; T.isnew = isnew;
                tri(ctx,&T);
                s = b; t = m;
                ipost = ANTI(s);
                apost = aux ? ANTI(t) : INT64_MAX;
                dgmin = 2*BUCK_WIDTH; dgmax = 0;
                ahgh  = -chain_break;
                alow  = (apost < ipost) ? apost : ipost;
                cov = 0; go = 1; mix = 0; nseed = 0;
                while (go)
                  { if (apost < ipost)
                      { lcp  = (int) get_bits(seeds+t,0,6);
                        dg   = (int) get_bits(seeds+t,6,6) + BUCK_WIDTH;
                        anti = apost;
                        t += 1;
                        apost = (t >= e) ? INT64_MAX : ANTI(t);
                        wch = 0x2;
                      }
                    else
                      { if (s < m)
                          { lcp = (int) get_bits(seeds+s,0,6);
                            dg  = (int) get_bits(seeds+s,6,6);
                          }
                        else
                          { lcp = 0; dg = 0; }       /* reference reads past the band: values unused */
                        anti = ipost;
                        s += 1;
                        if (s >= m)
                          { if (s > m) go = 0; else ipost = INT64_MAX; }
                        else
                          ipost = ANTI(s);
                        wch = 0x1;
                      }
                    lcp <<= 1;

                    if (anti < ahgh + chain_break)
                      { int64_t cps = anti + lcp;
                        if (cps > ahgh)
                          { if (anti >= ahgh) cov += lcp; else cov += (int) (cps-ahgh);
                            ahgh = cps;
                          }
                        mix |= wch;
                        if (dg < dgmin) dgmin = dg; else if (dg > dgmax) dgmax = dg;
                        nseed += 1;
                      }
                    else
                      { if (cov >= chain_min && (mix != 1 || isnew))
                          hit(ctx,&T,alow,ahgh,dgmin,dgmax,nseed);
                        if (go)
                          { cov = lcp; ahgh = anti + lcp; mix = wch; alow = anti;
                            dgmin = dgmax = dg; nseed = 1;
                          }
                      }
                  }
              }

            if (e >= g1) break;
            if (aux)
              { b = m; cdiag += 1; isnew = 0; }
            else
              { b = e;
                cdiag = BAND(e);
                while (e < g1 && BAND(e) == cdiag) e += 1;
                isnew = 1;
              }
          }
      }
      g0 = g1;
    }
#undef ANTI
#undef BAND
#undef GRP
}

/*  orc_search: every chain goes through the tube stepping and Local_Alignment calls of
    FastGA.c:3157-3340 as soon as the scan closes it; alast blocks within a triple.  */
typedef struct
  { const rec128 *seeds; const orc_layout *L; const orc_params *P; const orc_spec *spec;
    const int *perm1, *perm2; const char **aseq, **acseq, **bseq; const int64_t *alens, *blens;
    orc_result *R; orc_work *work; orc_path *path; int alnMin; double alnRate;
    orc_calllog *log;                       /* NULL (orc_search), or the call list of orc_search_calls */
    int comp, ctg1, ctg2; int64_t alen, blen, mlen, doffset, aoffset, alast; const char *as, *bs;
    int ngrp; uint64_t gkey;                /* align_contigs calls so far, (strand, contig pair) of the last */
  } search_ctx;

static void search_triple(void *v, const orc_triple *T)
{ search_ctx *S = (search_ctx *) v;
  const orc_layout *L = S->L;
  int p_jc = 12 + L->anti_bits + L->band_bits, p_ic = p_jc + L->jc_bits, p_cp = p_ic + L->ic_bits;
  const rec128 *r = S->seeds + T->b;
  if (S->ngrp == 0 || T->key != S->gkey)            /* one align_contigs call per (strand, contig pair) */
    { S->ngrp += 1; S->gkey = T->key; }
  S->comp = (int) get_bits(r,p_cp,1);
  S->ctg1 = S->perm1[get_bits(r,p_ic,L->ic_bits)];
  S->ctg2 = S->perm2[get_bits(r,p_jc,L->jc_bits)];
  S->alen = S->alens[S->ctg1]; S->blen = S->blens[S->ctg2]; S->mlen = S->alen + S->blen;
  S->doffset = S->alen - (L->amxpos + L->bmxpos); S->aoffset = S->alen - L->amxpos;
  S->as = S->comp ? S->acseq[S->ctg1] : S->aseq[S->ctg1];
  S->bs = S->bseq[S->ctg2];
  S->alast = -1;
}

static void log_call(orc_calllog *g, int comp, int ctg1, int ctg2, int low, int hgh, int anti, int lbord,
                     int hbord, int rec, const orc_path *p)
{ orc_call *c;
  if (g->ncall >= g->maxcall)
    { g->maxcall = g->maxcall*2 + 256;
      g->call = (orc_call *) realloc(g->call,sizeof(orc_call)*g->maxcall);
    }
  if (g->tlen + p->tlen > g->tmax)
    { g->tmax = (g->tlen + p->tlen)*2 + 4096;
      g->tpool = (uint8_t *) realloc(g->tpool,g->tmax);
    }
  c = g->call + g->ncall;
  c->comp = comp; c->ctg1 = ctg1; c->ctg2 = ctg2; c->low = low; c->hgh = hgh; c->anti = anti;
  c->lbord = lbord; c->hbord = hbord; c->rec = rec;
  c->abpos = p->abpos; c->bbpos = p->bbpos; c->aepos = p->aepos; c->bepos = p->bepos;
  c->diffs = p->diffs; c->tlen = p->tlen; c->pad = 0;
  c->pass0 = (int) g->npass; c->npass = 0;
  while (c->pass0 > 0 && g->pass[c->pass0-1].call == g->ncall) c->pass0 -= 1;
  c->npass = (int) g->npass - c->pass0;
  c->toff = g->tlen;
  memcpy(g->tpool+g->tlen,p->trace,p->tlen);
  g->tlen += p->tlen;
  g->ncall += 1;
}

static void search_hit(void *v, const orc_triple *T, int64_t alow, int64_t ahgh, int dgmin, int dgmax,
                       int64_t nseed)
{ search_ctx *S = (search_ctx *) v;
  orc_path *path = S->path;
  int comp = S->comp, ctg1 = S->ctg1, ctg2 = S->ctg2, alen = (int) S->alen, blen = (int) S->blen;
  int64_t amid, eant;
  (void) nseed;
  S->R->nhit += 1;
  dgmin += (int) (T->cdiag<<BUCK_SHIFT);
  dgmax += (int) (T->cdiag<<BUCK_SHIFT);
  if (comp)
    { dgmin += (int) S->doffset; dgmax += (int) S->doffset;
      alow += S->aoffset; ahgh += S->aoffset;
    }
  else
    { dgmin -= (int) S->L->bmxpos; dgmax -= (int) S->L->bmxpos; }

  if (ahgh > S->alast)
    { if (alow < S->alast) alow = S->alast;
      ahgh -= BUCK_ANTI;
      do
        { int rlen;
          amid = alow + BUCK_ANTI;
          if (amid > ahgh)
            { amid = ahgh;
              if (amid + dgmin < 0)
                { dgmin = (int) -amid;
                  if (dgmin > dgmax) break;
                }
            }
          int lbord = -1, hbord = -1, called = 1;
          if (g_self && ctg1 == ctg2 && !comp)
            { if (dgmin > 0)
                { lbord = dgmin-1; g_self_cnt[2] += 1; }
              else if (dgmax < 0)
                { hbord = -(dgmax+1); g_self_cnt[3] += 1; }
              else
                { path->abpos = path->aepos = 0; called = 0;
                  g_self_cnt[0] += 1;
                  if (path->bepos > alow) g_self_cnt[1] += 1;
                  if (g_straddle_zero) path->bbpos = path->bepos = 0;
                }
            }
          if (called)
            orc_local_alignment(S->work,S->spec,S->as,alen,S->bs,blen,comp,
                                dgmin,dgmax,(int) amid,lbord,hbord,path);
          rlen = path->aepos - path->abpos;
          if (called && S->log != NULL)
            log_call(S->log,comp,ctg1,ctg2,dgmin,dgmax,(int) amid,lbord,hbord,
                     rlen >= S->alnMin && S->alnRate*rlen >= path->diffs,path);
          if (rlen >= S->alnMin && S->alnRate*rlen >= path->diffs)
            { orc_ovl o;
              o.comp = comp; o.aread = ctg1; o.bread = ctg2;
              o.abpos = path->abpos; o.bbpos = path->bbpos;
              o.aepos = path->aepos; o.bepos = path->bepos;
              o.diffs = path->diffs; o.tlen = path->tlen; o.grp = S->ngrp-1; o.toff = 0;
              res_push(S->R,&o,path->trace);
            }
          if (comp) eant = S->mlen - (path->abpos + path->bbpos);
          else      eant = path->aepos + path->bepos;
          if (eant <= alow) alow = amid; else alow = eant;
        }
      while (alow < ahgh);
      S->alast = alow;
    }
}

static int64_t search(const rec128 *seeds, int64_t n, const orc_layout *L, const orc_params *P,
                      const orc_spec *spec, const int *perm1, const int *perm2,
                      const char **aseq, const char **acseq, const int64_t *alens,
                      const char **bseq, const int64_t *blens, orc_result *R, orc_calllog *log)
{ search_ctx S;
  orc_path path; memset(&path,0,sizeof(path));
  memset(&S,0,sizeof(S));
  S.seeds = seeds; S.L = L; S.P = P; S.spec = spec; S.perm1 = perm1; S.perm2 = perm2;
  S.aseq = aseq; S.acseq = acseq; S.bseq = bseq; S.alens = alens; S.blens = blens;
  S.R = R; S.work = orc_new_work(); S.path = &path;
  S.log = log; S.work->log = log;
  S.alnMin = P->align_min - 50;
  S.alnRate = P->align_rate + .05;
  memset(g_self_cnt,0,sizeof(g_self_cnt));
  chain_scan(seeds,n,L,P->chain_break,P->chain_min,search_triple,search_hit,&S);
  free(path.trace);
  orc_free_work(S.work);
  return R->novl;
}

int64_t orc_search(const rec128 *seeds, int64_t n, const orc_layout *L, const orc_params *P,
                   const orc_spec *spec, const int *perm1, const int *perm2,
                   const char **aseq, const char **acseq, const int64_t *alens,
                   const char **bseq, const int64_t *blens, orc_result *R)
{ return search(seeds,n,L,P,spec,perm1,perm2,aseq,acseq,alens,bseq,blens,R,NULL); }

/*  orc_search_calls: orc_search, and the list of its Local_Alignment calls with the passes of each
    (orc_calllog_* read it out; orc_free_calllog releases it).  */
orc_calllog *orc_new_calllog(void) { return (orc_calllog *) calloc(1,sizeof(orc_calllog)); }
void     orc_free_calllog(orc_calllog *g) { free(g->call); free(g->tpool); free(g->pass); free(g); }
int64_t  orc_calllog_calls(orc_calllog *g) { return g->ncall; }
int64_t  orc_calllog_passes(orc_calllog *g) { return g->npass; }
orc_call *orc_calllog_call(orc_calllog *g) { return g->call; }
orc_pass *orc_calllog_pass(orc_calllog *g) { return g->pass; }
uint8_t  *orc_calllog_traces(orc_calllog *g) { return g->tpool; }

int64_t orc_search_calls(const rec128 *seeds, int64_t n, const orc_layout *L, const orc_params *P,
                         const orc_spec *spec, const int *perm1, const int *perm2,
                         const char **aseq, const char **acseq, const int64_t *alens,
                         const char **bseq, const int64_t *blens, orc_result *R, orc_calllog *log)
{ return search(seeds,n,L,P,spec,perm1,perm2,aseq,acseq,alens,bseq,blens,R,log); }

/*  orc_chains: the chains alone.  trip gets 8 words per scanned triple (b, m, e, isnew, (strand,
    contig pair) key, cdiag, first hit, hits), hits 5 words per chain (alow, ahgh, dgmin, dgmax,
    seeds); counts = (triples, chains).  With trip or hits NULL only the counts are made.  */
typedef struct { int64_t *trip, *hits, ntrip, nhit; } chains_ctx;

static void chains_triple(void *v, const orc_triple *T)
{ chains_ctx *C = (chains_ctx *) v;
  if (C->trip != NULL)
    { int64_t *t = C->trip + 8*C->ntrip;
      t[0] = T->b; t[1] = T->m; t[2] = T->e; t[3] = T->isnew; t[4] = (int64_t) T->key; t[5] = T->cdiag;
      t[6] = C->nhit; t[7] = 0;
    }
  C->ntrip += 1;
}

static void chains_hit(void *v, const orc_triple *T, int64_t alow, int64_t ahgh, int dgmin, int dgmax,
                       int64_t nseed)
{ chains_ctx *C = (chains_ctx *) v;
  (void) T;
  if (C->hits != NULL && C->trip != NULL)
    { int64_t *h = C->hits + 5*C->nhit;
      h[0] = alow; h[1] = ahgh; h[2] = dgmin; h[3] = dgmax; h[4] = nseed;
      C->trip[8*(C->ntrip-1) + 7] += 1;
    }
  C->nhit += 1;
}

void orc_chains(const rec128 *seeds, int64_t n, const orc_layout *L, int chain_break, int chain_min,
                int64_t *trip, int64_t *hits, int64_t *counts)
{ chains_ctx C;
  C.trip = trip; C.hits = hits; C.ntrip = 0; C.nhit = 0;
  if (trip == NULL || hits == NULL) C.trip = C.hits = NULL;
  chain_scan(seeds,n,L,chain_break,chain_min,chains_triple,chains_hit,&C);
  counts[0] = C.ntrip; counts[1] = C.nhit;
}

/***********************************************************************************************
 *  F.  Redundancy filter of align_contigs (FastGA.c:3405-3685) with entwine (:2818-2941), run on
 *      the records of each align_contigs call, then the SORT_MAP order of la_sort (:3800-3835)
 *      over every survivor.
 *
 *  Restated from the reference's rules, not from fastga_b200/csrc/filter.cu: entwine keeps the
 *  running separation closest to zero and the last meeting point, the sweeps walk a pointer array
 *  in libc qsort order, every record carries ELIMINATED / OWNS_TRACE flags, and each fusion cuts
 *  a fresh trace at the meeting point.  orc_filter_counters reads, per outcome, how often the last
 *  orc_filter went through each branch (FC_* below).
 **********************************************************************************************/

#define F_TSPACE      100
#define F_BOX_FUZZ     10
#define F_ELIMINATED  0x1
#define F_OWNS_TRACE  0x2

typedef struct
  { orc_ovl  o;             /* o.toff unused */
    uint8_t *trace;         /* (diffs, B-advance) byte pairs */
    int      flags;
    int64_t  pos;           /* place in the filter's output stream: the reference's address order */
  } fl_rec;

enum { FC_S1_BOTH_KEEP_O,   /* sweep 1: same start and end, o kept (o.diffs < w.aepos) */
       FC_S1_BOTH_DROP_O,   /*          same start and end, o dropped */
       FC_S1_START_KEEP_O,  /*          same start only, o ends later */
       FC_S1_START_DROP_O,  /*          same start only, w ends at or after o */
       FC_S1_END_KEEP_O,    /*          same end only, o starts earlier */
       FC_S1_END_DROP_O,    /*          same end only, o starts at or after w */
       FC_S2_B_DISJOINT,    /* sweep 2: B-intervals apart, w skipped */
       FC_S2_FUSE,          /*          paths meet: o continues as w (every fusion) */
       FC_S2_FUSE_DEAD_O,   /*          ... into an o that its row has already eliminated */
       FC_S2_FUSE_W_OWNS,   /*          ... with a w that already owns a fused trace */
       FC_S2_BOX_DROP_W,    /*          paths apart, w inside o's box */
       FC_S2_BOX_DROP_O,    /*          paths apart, o inside w's box */
       FC_S2_APART_KEPT,    /*          paths apart, neither box inside the other */
       FC_S2_CROSS,         /*          paths touch or cross without a meeting point: no action */
       FC_S2_ROW_EXTENDED,  /*          a w visited only because a fusion moved o's end */
       FC_N };

static int64_t g_filter_cnt[FC_N];
void orc_filter_counters(int64_t *out) { memcpy(out,g_filter_cnt,sizeof(g_filter_cnt)); }

/* min tracks the separation closest to zero; it sticks at 0 once two separations differ in sign
   or one is 0 (FastGA.c:2876-2887) */
static int closer(int min, int d)
{ if (min < 0 && d > min)
    return (d >= 0 ? 0 : d);
  if (min > 0 && d < min)
    return (d <= 0 ? 0 : d);
  return (min);
}

/* J starts at or before K on A.  The B-separation K - J at K's start (J interpolated inside its
   interval), at every trace point both paths pass strictly before the first end, and at that end
   (the path that does not end there interpolated from the trace point before it).  Returns the
   separation closest to zero (0: the paths touch or cross); *where is the last of those trace
   points at separation 0, -1 if there is none (FastGA.c:2818-2941). */
static int entwine(const orc_ovl *J, const uint8_t *jtr, const orc_ovl *K, const uint8_t *ktr, int *where)
{ int ac, ae, y2, b2, yp, i, j, k, min;

  *where = -1;
  y2 = J->bbpos;
  b2 = K->bbpos;
  ac = (K->abpos/F_TSPACE)*F_TSPACE;
  j  = 1 + 2*(K->abpos/F_TSPACE - J->abpos/F_TSPACE);
  for (i = 1; i < j; i += 2)
    y2 += jtr[i];
  if (j == 1)
    yp = y2 + (jtr[j] * (K->abpos - J->abpos)) / (ac+F_TSPACE - J->abpos);
  else
    yp = y2 + (jtr[j] * (K->abpos - ac)) / F_TSPACE;
  min = b2-yp;

  ae = (J->aepos < K->aepos) ? J->aepos : K->aepos;
  for (k = 1, ac += F_TSPACE; ac < ae; ac += F_TSPACE, j += 2, k += 2)
    { y2 += jtr[j];
      b2 += ktr[k];
      i = b2-y2;
      min = closer(min,i);
      if (i == 0)
        *where = ac;
    }
  ac -= F_TSPACE;

  if (ae == J->aepos)
    { y2 = J->bepos;
      if (K->aepos >= ac)
        b2 += (ktr[k] * (ae-ac)) / F_TSPACE;
      else
        b2 += (ktr[k] * (ae-ac)) / (K->aepos-ac);
    }
  else
    { b2 = K->bepos;
      if (J->aepos >= ac)
        y2 += (jtr[j] * (ae-ac)) / F_TSPACE;
      else
        y2 += (jtr[j] * (ae-ac)) / (J->aepos-ac);
    }
  return (closer(min,b2-y2));
}

static int FL_ASORT(const void *l, const void *r)      /* FastGA.c:2962 */
{ return ((*(fl_rec **) l)->o.abpos - (*(fl_rec **) r)->o.abpos); }

/* o continues as w from the trace point `where` on: o's intervals up to it, then w's after it */
static void fuse(fl_rec *o, const fl_rec *w, int where)
{ orc_ovl *op = &o->o;
  const orc_ovl *wp = &w->o;
  int ocut = 2*(((where - op->abpos)-1)/F_TSPACE + 1);
  int wcut = 2*(((where - wp->abpos)-1)/F_TSPACE + 1);
  int tlen = ocut + (wp->tlen - wcut), d = 0, g, h = 0;
  uint8_t *nt = (uint8_t *) malloc(tlen > 0 ? tlen : 1);

  for (g = 0; g < ocut; g += 2, h += 2)
    { d += (nt[h] = o->trace[g]); nt[h+1] = o->trace[g+1]; }
  for (g = wcut; g < wp->tlen; g += 2, h += 2)
    { d += (nt[h] = w->trace[g]); nt[h+1] = w->trace[g+1]; }
  if (o->flags & F_OWNS_TRACE)
    free(o->trace);
  o->trace  = nt;
  o->flags |= F_OWNS_TRACE;
  op->tlen  = tlen;
  op->diffs = d;
  op->aepos = wp->aepos;
  op->bepos = wp->bepos;
}

/* the redundancy filter of one align_contigs call on perm[0..n) */
static void filter_call(fl_rec **perm, int n)
{ int j, k, where, dist;

  qsort(perm,n,sizeof(fl_rec *),FL_ASORT);

  //  Sweep 1: equal start points or equal end points

  for (j = n-1; j >= 0; j--)
    { fl_rec  *o  = perm[j];
      orc_ovl *op = &o->o;
      for (k = j+1; k < n; k++)
        { fl_rec  *w  = perm[k];
          orc_ovl *wp = &w->o;
          int      same_start, same_end, drop_o;

          if (op->aepos <= wp->abpos)
            break;
          if (w->flags & F_ELIMINATED)
            continue;
          same_start = (op->abpos == wp->abpos && op->bbpos == wp->bbpos);
          same_end   = (op->aepos == wp->aepos && op->bepos == wp->bepos);
          if (same_start && same_end)
            { drop_o = !(op->diffs < wp->aepos);          /* diffs against aepos, as FastGA.c:3456 */
              g_filter_cnt[drop_o ? FC_S1_BOTH_DROP_O : FC_S1_BOTH_KEEP_O] += 1;
            }
          else if (same_start)
            { drop_o = !(op->aepos > wp->aepos);
              g_filter_cnt[drop_o ? FC_S1_START_DROP_O : FC_S1_START_KEEP_O] += 1;
            }
          else if (same_end)
            { drop_o = !(op->abpos < wp->abpos);
              g_filter_cnt[drop_o ? FC_S1_END_DROP_O : FC_S1_END_KEEP_O] += 1;
            }
          else
            continue;
          if (drop_o)
            { o->flags |= F_ELIMINATED;
              break;
            }
          w->flags |= F_ELIMINATED;
        }
    }

  //  Sweep 2: paths that meet are fused, a path apart from and boxed in by another is dropped

  for (j = n-1; j >= 0; j--)
    { fl_rec  *o  = perm[j];
      orc_ovl *op = &o->o;
      int      aend0 = op->aepos;

      if (o->flags & F_ELIMINATED)
        continue;
      for (k = j+1; k < n; k++)
        { fl_rec  *w  = perm[k];
          orc_ovl *wp = &w->o;

          if (op->aepos <= wp->abpos)                   /* o's end is re-read: a fusion moves it */
            break;
          if (w->flags & F_ELIMINATED)
            continue;
          if (wp->abpos >= aend0)
            g_filter_cnt[FC_S2_ROW_EXTENDED] += 1;
          if (op->bepos <= wp->bbpos || op->bbpos >= wp->bepos)
            { g_filter_cnt[FC_S2_B_DISJOINT] += 1;
              continue;
            }

          dist = entwine(op,o->trace,wp,w->trace,&where);
          if (where != -1)
            { g_filter_cnt[FC_S2_FUSE] += 1;
              if (o->flags & F_ELIMINATED)
                g_filter_cnt[FC_S2_FUSE_DEAD_O] += 1;
              if (w->flags & F_OWNS_TRACE)
                g_filter_cnt[FC_S2_FUSE_W_OWNS] += 1;
              fuse(o,w,where);
              w->flags |= F_ELIMINATED;
              continue;
            }
          if (dist == 0)
            { g_filter_cnt[FC_S2_CROSS] += 1;
              continue;
            }
          if ((op->aepos - op->abpos) + F_BOX_FUZZ >= wp->aepos - wp->abpos)
            { if (wp->aepos <= op->aepos + F_BOX_FUZZ && wp->bbpos >= op->bbpos - F_BOX_FUZZ &&
                  wp->bepos <= op->bepos + F_BOX_FUZZ)
                { g_filter_cnt[FC_S2_BOX_DROP_W] += 1;
                  w->flags |= F_ELIMINATED;
                  continue;
                }
            }
          else
            { if (op->aepos <= wp->aepos + F_BOX_FUZZ && op->bbpos >= wp->bbpos - F_BOX_FUZZ &&
                  op->bepos <= wp->bepos + F_BOX_FUZZ && op->abpos >= wp->abpos - F_BOX_FUZZ)
                { g_filter_cnt[FC_S2_BOX_DROP_O] += 1;
                  o->flags |= F_ELIMINATED;              /* o still finishes its row */
                  continue;
                }
            }
          g_filter_cnt[FC_S2_APART_KEPT] += 1;
        }
    }
}

static int SORT_MAP(const void *x, const void *y)     /* FastGA.c:3800-3835, position for address */
{ const fl_rec *l = *(fl_rec **) x;
  const fl_rec *r = *(fl_rec **) y;

  if (l->o.aread != r->o.aread)
    return (l->o.aread - r->o.aread);
  if (l->o.abpos != r->o.abpos)
    return (l->o.abpos - r->o.abpos);
  if (l->o.bread != r->o.bread)
    return (l->o.bread - r->o.bread);
  if (l->o.comp != r->o.comp)
    return (l->o.comp - r->o.comp);
  return ((l->pos > r->pos) - (l->pos < r->pos));
}

/*  orc_filter: in[0..n) are raw alignments in discovery order (traces at tpool + in[i].toff), and
    every run of equal in[i].grp is the output of one align_contigs call.  Filters each call
    (do_filter = 0: keeps every record), writes the survivors of each call in sweep order one call
    after the other, and returns them in R in SORT_MAP order, ties by that position.  */
int64_t orc_filter(const orc_ovl *in, int64_t n, const uint8_t *tpool, int do_filter, orc_result *R)
{ fl_rec  *rec  = (fl_rec *) malloc(sizeof(fl_rec)*(n > 0 ? n : 1));
  fl_rec **perm = (fl_rec **) malloc(sizeof(fl_rec *)*(n > 0 ? n : 1));
  fl_rec **live = (fl_rec **) malloc(sizeof(fl_rec *)*(n > 0 ? n : 1));
  int64_t  i, b, e, nlive = 0;

  memset(g_filter_cnt,0,sizeof(g_filter_cnt));
  for (i = 0; i < n; i++)
    { rec[i].o = in[i];
      rec[i].trace = (uint8_t *) tpool + in[i].toff;
      rec[i].flags = 0;
      rec[i].pos = -1;
    }
  for (b = 0; b < n; b = e)
    { for (e = b; e < n && in[e].grp == in[b].grp; e++)
        perm[e-b] = rec+e;
      if (do_filter)
        filter_call(perm,(int) (e-b));
      for (i = 0; i < e-b; i++)
        if ((perm[i]->flags & F_ELIMINATED) == 0)
          { perm[i]->pos = nlive;
            live[nlive++] = perm[i];
          }
    }

  qsort(live,nlive,sizeof(fl_rec *),SORT_MAP);
  for (i = 0; i < nlive; i++)
    res_push(R,&live[i]->o,live[i]->trace);

  for (i = 0; i < n; i++)
    if (rec[i].flags & F_OWNS_TRACE)
      free(rec[i].trace);
  free(live);
  free(perm);
  free(rec);
  return (nlive);
}
