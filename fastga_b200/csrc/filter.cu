// Host side of the path after the kernels: the redundancy filter of align_contigs and the final
// (aread, abpos, bread, comp) ordering.  Stays host C++ on purpose (SURVEY 2: "stays host C; must
// be bit-compatible"): it is <1 % of the work, is driven by libc qsort's tie order, and works on
// the few hundred thousand records the device returns.  A host that prefers the reference's own
// filter takes the raw, discovery-ordered records of fgb_extend instead (INTEGRATION.md).
//
// Replaces (reference file:line):
//   entwine                         FastGA.c:2818-2941
//   redundancy filter               FastGA.c:3407-3685   (per (A-contig, B-contig, strand) call)
//   la_sort / SORT_MAP order        FastGA.c:3800-3900
#include "stages.h"
#include "handles.h"
#include <stdlib.h>
#include <string.h>
#include <vector>
#include <algorithm>

#define TSPACE    100
#define BOX_FUZZ  10

//  The rules below are the reference's (their result is part of the .1aln contract, libc qsort tie
//  order and the `diffs < aepos` comparison of FastGA.c:3456 included); the implementation is this
//  repo's own: paths are compared by sampling both on the common trace-point grid and reducing the
//  separations, the group lives in one array in sweep order, and the two sweeps share one driver.

namespace {

struct Aln                                   // one local alignment of a (A-contig, B-contig, strand) group
{ int ab, bb, ae, be, diffs, tlen;
  const unsigned char *trace;                // (diffs, B-advance) byte pairs, one per trace interval
  std::vector<unsigned char> spliced;        // backing store once two alignments have been fused
  bool dead;
  int bstep(int i) const { return trace[2*i+1]; }
};

int by_abpos(const void *l, const void *r)   // the comparator of FastGA.c:2962 on the same libc qsort
{ return (*(Aln * const *) l)->ab - (*(Aln * const *) r)->ab; }

struct Braid { bool apart; int meet; };      // apart: the paths never touch; meet: last shared trace point, -1 if none

//  J starts at or before K on A.  Both paths are sampled at K's start, at every trace point they
//  share, and at the end of the shorter one (linear interpolation inside a trace interval with the
//  reference's integer arithmetic, FastGA.c:2818-2941); `apart` iff every separation has one sign.
Braid braid(const Aln &J, const Aln &K)
{ const int g0 = (K.ab / TSPACE) * TSPACE;                 // trace point at or before K's start
  const int skip = K.ab / TSPACE - J.ab / TSPACE;          // whole intervals of J before it
  int yj = J.bb;
  for (int u = 0; u < skip; u++) yj += J.bstep(u);
  const int from = skip ? g0 : J.ab, span = skip ? TSPACE : g0 + TSPACE - J.ab;
  int sep = K.bb - (yj + J.bstep(skip) * (K.ab - from) / span);
  int lo = sep, hi = sep, meet = -1, yk = K.bb, t = 0;
  const int end = J.ae < K.ae ? J.ae : K.ae;
  for (int g = g0 + TSPACE; g < end; g += TSPACE, t++)
    { yj += J.bstep(skip + t);
      yk += K.bstep(t);
      sep = yk - yj;
      if (sep < lo) lo = sep;
      if (sep > hi) hi = sep;
      if (sep == 0) meet = g;
    }
  const int rest = end - (g0 + t*TSPACE);                  // into the last, partial interval
  if (end == J.ae) { yj = J.be; yk += K.bstep(t) * rest / TSPACE; }
  else             { yk = K.be; yj += J.bstep(skip + t) * rest / TSPACE; }
  sep = yk - yj;
  if (sep < lo) lo = sep;
  if (sep > hi) hi = sep;
  Braid r; r.apart = (lo > 0 || hi < 0); r.meet = meet;
  return r;
}

inline int intervals_to(const Aln &p, int apoint)          // trace intervals of p covering [p.ab, apoint]
{ return (apoint - p.ab + TSPACE - 1) / TSPACE; }

//  o keeps its head up to the shared trace point and continues as w (FastGA.c:3524-3569)
void splice(Aln &o, const Aln &w, int at)
{ const int ocut = 2*intervals_to(o,at), wcut = 2*intervals_to(w,at);
  std::vector<unsigned char> t;
  t.reserve(ocut + (w.tlen > wcut ? w.tlen - wcut : 0));
  t.insert(t.end(),o.trace,o.trace + ocut);
  if (w.tlen > wcut) t.insert(t.end(),w.trace + wcut,w.trace + w.tlen);
  int d = 0;
  for (size_t q = 0; q < t.size(); q += 2) d += t[q];
  o.spliced.swap(t);
  o.trace = o.spliced.data();
  o.tlen  = (int) o.spliced.size();
  o.diffs = d;
  o.ae = w.ae; o.be = w.be;
}

inline bool inside(const Aln &in, const Aln &out, bool also_start)   // box test with BOX_FUZZ slack (:3571-3587)
{ return in.ae <= out.ae + BOX_FUZZ && in.bb >= out.bb - BOX_FUZZ && in.be <= out.be + BOX_FUZZ &&
         (!also_start || in.ab >= out.ab - BOX_FUZZ);
}

//  Visits, for every alignment o from the last to the first of the sweep order, the later
//  alignments w whose A-interval starts before o (currently) ends.  rule(o,w) returns false to
//  leave o's row early.
template<class Rule> void sweep(std::vector<Aln *> &row, bool live_o_only, Rule rule)
{ const int n = (int) row.size();
  for (int j = n-1; j >= 0; j--)
    { Aln &o = *row[j];
      if (live_o_only && o.dead) continue;
      for (int k = j+1; k < n && o.ae > row[k]->ab; k++)
        if (!row[k]->dead && !rule(o,*row[k])) break;
    }
}

void filter_group(std::vector<Aln> &g)
{ std::vector<Aln *> row(g.size());
  for (size_t i = 0; i < g.size(); i++) row[i] = &g[i];
  qsort(row.data(),row.size(),sizeof(Aln *),by_abpos);     // libc: its tie order is part of the result (:3435)

  //  sweep 1: two alignments with the same start point, or the same end point, are one finding
  sweep(row,false,[](Aln &o, Aln &w)
    { const bool start = (o.ab == w.ab && o.bb == w.bb), stop = (o.ae == w.ae && o.be == w.be);
      if (!start && !stop) return true;
      bool keep_o;
      if (start && stop) keep_o = o.diffs < w.ae;          // sic: diffs against aepos (FastGA.c:3456)
      else if (start)    keep_o = o.ae > w.ae;             // the longer one survives
      else               keep_o = o.ab < w.ab;
      (keep_o ? w : o).dead = true;
      return keep_o;                                       // a dead o stops looking
    });

  //  sweep 2: overlapping boxes -- fuse at a shared trace point, else drop a contained box
  sweep(row,true,[](Aln &o, Aln &w)
    { if (o.be <= w.bb || o.bb >= w.be) return true;       // B-intervals apart
      const Braid x = braid(o,w);
      if (x.meet >= 0) { splice(o,w,x.meet); w.dead = true; }
      else if (x.apart)
        { if ((o.ae - o.ab) + BOX_FUZZ >= w.ae - w.ab) { if (inside(w,o,false)) w.dead = true; }
          else if (inside(o,w,true)) o.dead = true;        // o, though dead, finishes its row (:3583)
        }
      return true;
    });

  std::vector<Aln> kept;                                   // survivors in sweep order (:3649-3680)
  for (Aln *p : row) if (!p->dead) kept.push_back(std::move(*p));
  for (Aln &k : kept) if (!k.spliced.empty()) k.trace = k.spliced.data();
  g.swap(kept);
}

}  // namespace

struct fgb_alns
{ long long n = 0, nraw = 0;
  std::vector<int> fields;                  // n x 9: comp aread bread abpos bbpos aepos bepos diffs tlen
  std::vector<long long> toff;
  std::vector<unsigned char> pool;
};

struct RawRef { int triple, seq; long long off; };

//  Raw device records -> discovery order -> per contig-pair filter -> final SORT_MAP order.
//  perm1/perm2 map contig ranks (seed records) to original contig numbers (FastGA.c:3007-3008).

extern "C" int fgb_filter(const fgb_overlaps *O, const int *perm1, const int *perm2, int jc_bits,
                          int ic_bits, int do_filter, fgb_alns **out)
{ long long nb = fgb_overlaps_bytes(O);
  const unsigned char *buf = fgb_overlaps_data(O);
  std::vector<RawRef> refs;
  for (long long off = 0; off < nb; )
    { const ovl_hdr *h = (const ovl_hdr *) (buf + off);
      RawRef r; r.triple = h->triple; r.seq = h->seq; r.off = off;
      refs.push_back(r);
      off += ovl_bytes(h->tlen);
    }
  std::sort(refs.begin(),refs.end(),[](const RawRef &a, const RawRef &b)
            { return a.triple != b.triple ? a.triple < b.triple : a.seq < b.seq; });

  fgb_alns *R = new fgb_alns();
  R->nraw = (long long) refs.size();
  struct Fin { int comp, aread, bread; Aln o; };
  std::vector<Fin> fin;
  size_t i = 0;
  while (i < refs.size())
    { int pk = ((const ovl_hdr *) (buf + refs[i].off))->pairkey;
      std::vector<Aln> g;
      size_t e = i;
      while (e < refs.size() && ((const ovl_hdr *) (buf + refs[e].off))->pairkey == pk)
        { const ovl_hdr *h = (const ovl_hdr *) (buf + refs[e].off);
          Aln o;
          o.ab = h->abpos; o.bb = h->bbpos; o.ae = h->aepos; o.be = h->bepos; o.diffs = h->diffs; o.tlen = h->tlen;
          o.dead = false;
          o.trace = buf + refs[e].off + sizeof(ovl_hdr);
          g.push_back(std::move(o));
          e += 1;
        }
      if (do_filter) filter_group(g);
      int jc = pk & ((1 << jc_bits) - 1), ic = (pk >> jc_bits) & ((1 << ic_bits) - 1);
      int comp = (pk >> (jc_bits + ic_bits)) & 1;
      for (size_t q = 0; q < g.size(); q++)
        { Fin f; f.comp = comp; f.aread = perm1[ic]; f.bread = perm2[jc]; f.o = std::move(g[q]);
          fin.push_back(std::move(f));
          if (!fin.back().o.spliced.empty()) fin.back().o.trace = fin.back().o.spliced.data();
        }
      i = e;
    }

  //  SORT_MAP (FastGA.c:3800-3836): (aread, abpos, bread, comp); remaining ties by address in
  //  the reference (= order of arrival in its per-thread file) -> here stable order of arrival.
  std::vector<int> ord(fin.size());
  for (size_t q = 0; q < fin.size(); q++) ord[q] = (int) q;
  std::stable_sort(ord.begin(),ord.end(),[&](int a, int b)
    { const Fin &x = fin[a], &y = fin[b];
      if (x.aread != y.aread) return x.aread < y.aread;
      if (x.o.ab != y.o.ab) return x.o.ab < y.o.ab;
      if (x.bread != y.bread) return x.bread < y.bread;
      return x.comp < y.comp;
    });
  R->n = (long long) fin.size();
  R->fields.resize(R->n * 9);
  R->toff.resize(R->n);
  for (size_t q = 0; q < fin.size(); q++)
    { const Fin &f = fin[ord[q]];
      int *d = &R->fields[q*9];
      d[0] = f.comp; d[1] = f.aread; d[2] = f.bread;
      d[3] = f.o.ab; d[4] = f.o.bb; d[5] = f.o.ae; d[6] = f.o.be;
      d[7] = f.o.diffs; d[8] = f.o.tlen;
      R->toff[q] = (long long) R->pool.size();
      R->pool.insert(R->pool.end(),f.o.trace,f.o.trace + f.o.tlen);
    }
  *out = R;
  return FGB_OK;
}

extern "C" void fgb_alns_free(fgb_alns *a) { delete a; }
extern "C" long long fgb_alns_count(const fgb_alns *a) { return a->n; }
extern "C" long long fgb_alns_raw_count(const fgb_alns *a) { return a->nraw; }
extern "C" long long fgb_alns_pool_bytes(const fgb_alns *a) { return (long long) a->pool.size(); }
extern "C" int fgb_alns_get(const fgb_alns *a, int *fields /* n x 9 */, long long *toff,
                            unsigned char *pool)
{ memcpy(fields,a->fields.data(),sizeof(int)*a->fields.size());
  memcpy(toff,a->toff.data(),sizeof(long long)*a->toff.size());
  if (!a->pool.empty()) memcpy(pool,a->pool.data(),a->pool.size());
  return FGB_OK;
}
