// C-ABI of libfastga_b200.so: opaque handles (genome / GIX / seed set) over device memory and the
// host-buffer entry points the reference-side host code binds (see include/fastga_b200.h and
// INTEGRATION.md).  No torch types, no CPU fallback: every call runs the sm_90a kernels.
#include "stages.h"
#include "handles.h"
#include <vector>
#include <algorithm>
#include <string.h>
#include <chrono>

typedef unsigned long long u64;

static inline long long now_us()
{ return std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

static fgb_timings g_timings;

struct stage_timer
{ cudaEvent_t a, b; cudaStream_t st; float *dst;
  stage_timer(float *d, cudaStream_t s) : st(s), dst(d)
    { cudaEventCreate(&a); cudaEventCreate(&b); cudaEventRecord(a,st); }
  ~stage_timer()
    { cudaEventRecord(b,st); cudaEventSynchronize(b);
      float ms = 0; cudaEventElapsedTime(&ms,a,b); *dst += ms;
      cudaEventDestroy(a); cudaEventDestroy(b);
    }
};

//  A stage timer that does not wait: its events are read at the next host wait (fgb_stream_wait), or when the
//  timings are fetched.
struct lazy_event { cudaEvent_t a, b; float *dst; };
static std::vector<lazy_event> g_lazy;
static long long g_waits;

struct lazy_timer
{ lazy_event e; cudaStream_t st;
  lazy_timer(float *d, cudaStream_t s) : st(s)
    { e.dst = d; cudaEventCreate(&e.a); cudaEventCreate(&e.b); cudaEventRecord(e.a,st); }
  ~lazy_timer() { cudaEventRecord(e.b,st); g_lazy.push_back(e); }
};

//  adds the elapsed time of every timer whose end has been reached (wait = true: of every timer)
static void lazy_flush(bool wait)
{ size_t k = 0;
  for (const lazy_event &e : g_lazy)
    { if (wait) cudaEventSynchronize(e.b);
      else if (cudaEventQuery(e.b) != cudaSuccess) { g_lazy[k++] = e; continue; }
      float ms = 0;
      cudaEventElapsedTime(&ms,e.a,e.b);
      *e.dst += ms;
      cudaEventDestroy(e.a); cudaEventDestroy(e.b);
    }
  cudaGetLastError();
  g_lazy.resize(k);
}

//  The host waits of the k-mer table builds: each one counted (fgb_host_waits; the fused path reports the waits of
//  its table builds as fgb_run_stats.gix_waits).
cudaError_t fgb_stream_wait(cudaStream_t st)
{ g_waits += 1;
  cudaError_t e = cudaStreamSynchronize(st);
  lazy_flush(false);
  return e;
}

extern "C" long long fgb_host_waits() { return g_waits; }

void fgb_timing_add(int which, float ms)
{ if (which == 0) g_timings.triples_ms += ms;
  else if (which == 1) { g_timings.extend_ms += ms; g_timings.extend_launches += 1; }
  else if (which == 3) { g_timings.merge_ms += ms; g_timings.merge_launches += 1; }
  else g_timings.d2h_ms += ms;
}

void fgb_count_launch(int n) { g_timings.launches += n; }

//  Device memory for the stages comes from a process-wide caching allocator: blocks are rounded
//  to size classes, kept on a free list when released and handed out again on the next step, so
//  the steady state of a repeated workload makes no cudaMalloc/cudaFree calls at all (both stall
//  the device; the stream-ordered pool turned out to take 1-800 ms for the multi-GB arenas).
//  All work of a call is issued on one stream, so reuse after release is stream-ordered.

#include <map>
#include <unordered_map>
#include <mutex>

static std::multimap<size_t,void *> g_free;
static std::unordered_map<void *,size_t> g_live;
static std::mutex g_mem_lock;

static size_t size_class(size_t b)
{ if (b < 4096) return 4096;
  size_t p = 4096;
  while (p < b) p <<= 1;                 // p/2 < b <= p
  size_t step = p >> 4;                  // 8 classes per octave
  return ((b + step - 1) / step) * step;
}

cudaError_t fgb_dmalloc(void **p, size_t bytes, cudaStream_t st)
{ (void) st;
  size_t c = size_class(bytes);
  std::lock_guard<std::mutex> g(g_mem_lock);
  auto it = g_free.lower_bound(c);
  if (it != g_free.end() && it->first <= c + (c >> 2))
    { *p = it->second;
      g_live[*p] = it->first;
      g_free.erase(it);
      return cudaSuccess;
    }
  cudaError_t e = cudaMalloc(p,c);
  if (e != cudaSuccess)                  // out of memory: drop the cache and retry once
    { cudaGetLastError();
      for (auto &kv : g_free) cudaFree(kv.second);
      g_free.clear();
      e = cudaMalloc(p,c);
      if (e != cudaSuccess) return e;
    }
  g_live[*p] = c;
  return cudaSuccess;
}

void fgb_dfree(void *p, cudaStream_t st)
{ (void) st;
  if (p == NULL) return;
  std::lock_guard<std::mutex> g(g_mem_lock);
  auto it = g_live.find(p);
  if (it == g_live.end()) { cudaFree(p); return; }
  g_free.insert(std::make_pair(it->second,p));
  g_live.erase(it);
}

//  Gives every cached block back to the driver.
extern "C" void fgb_release_cache()
{ std::lock_guard<std::mutex> g(g_mem_lock);
  for (auto &kv : g_free) cudaFree(kv.second);
  g_free.clear();
}

//  Blocks of the cache handed to the caller (the sharded path's exchange buffers).
extern "C" int fgb_device_alloc(long long bytes, void **out, void *stream)
{ CUDA_TRY(fgb_dmalloc(out,(size_t) (bytes > 0 ? bytes : 16),(cudaStream_t) stream)); return FGB_OK; }
extern "C" void fgb_device_free(void *p) { fgb_dfree(p,0); }

//  Bytes of the blocks handed out and not yet given back (size classes, as the cache counts them).
extern "C" long long fgb_device_live_bytes()
{ std::lock_guard<std::mutex> g(g_mem_lock);
  long long s = 0;
  for (auto &kv : g_live) s += (long long) kv.second;
  return s;
}

extern "C" void fgb_timings_reset() { lazy_flush(true); memset(&g_timings,0,sizeof(g_timings)); }
extern "C" void fgb_timings_get(fgb_timings *out) { lazy_flush(true); *out = g_timings; }

/***********************************************************************************************
 *  Genome: the GDB as the path sees it (GDB.h:28-34 GDB_CONTIG {clen, boff} + the .bps image)
 **********************************************************************************************/

static const long long *g_sort_len;
static int LSORT(const void *l, const void *r)          // GIXmake.c:1628-1633: decreasing length
{ int x = *((const int *) l), y = *((const int *) r);
  return (int) (g_sort_len[y] - g_sort_len[x]);
}

extern "C" int fgb_genome_create(const unsigned char *bps, long long bps_bytes, int ncontig,
                                 const long long *clen, const long long *boff, int want_revcomp,
                                 fgb_genome **out, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (ncontig <= 0 || ncontig > 0x7fff) return FGB_ERR_LIMIT;   // contig rank is a 15-bit field
  std::unique_ptr<fgb_genome> g(new fgb_genome());
  g->ncontig = ncontig;
  g->clen.assign(clen,clen+ncontig);
  g->boff.assign(boff,boff+ncontig);
  g->woff.resize(ncontig+1);
  g->seqtot = 0; g->maxlen = 0;
  long long w = 2;                             // 16 zero bytes ahead of the first contig too
  for (int c = 0; c < ncontig; c++)
    { if (clen[c] >= 0x7fffffffll) return FGB_ERR_LIMIT;
      g->woff[c] = w;
      w += ((clen[c] + 31) >> 5) + 2;          // zero pad so 64-bit window reads stay inside
      w = (w + 1) & ~1ll;                      // 16-byte alignment of every contig
      g->seqtot += clen[c];
      if (clen[c] > g->maxlen) g->maxlen = clen[c];
    }
  g->woff[ncontig] = w;
  g->total_words = w;

  g->perm.resize(ncontig); g->crank.resize(ncontig);
  for (int c = 0; c < ncontig; c++) g->perm[c] = c;
  g_sort_len = clen;
  qsort(g->perm.data(),ncontig,sizeof(int),LSORT);     // same libc call as GIXmake.c:1959
  for (int c = 0; c < ncontig; c++) g->crank[g->perm[c]] = c;

  dblock<unsigned char> d_bps;
  dblock<long long> d_boff;
  CUDA_TRY(d_bps.alloc(bps_bytes + 16,st));
  CUDA_TRY(d_boff.alloc(ncontig,st));
  CUDA_TRY(g->d_clen.alloc(ncontig,st));
  CUDA_TRY(g->d_woff.alloc(ncontig+1,st));
  CUDA_TRY(g->d_crank.alloc(ncontig,st));
  CUDA_TRY(g->d_perm.alloc(ncontig,st));
  CUDA_TRY(g->d_seq.alloc(w + 1024,st));      // slack: the extension stages 1 KB tiles that may start near a contig end
  if (want_revcomp) CUDA_TRY(g->d_rseq.alloc(w + 1024,st));
  { stage_timer t(&g_timings.h2d_ms,st);
    CUDA_TRY(cudaMemcpyAsync(d_bps,bps,bps_bytes,cudaMemcpyHostToDevice,st));
    CUDA_TRY(cudaMemcpyAsync(d_boff,boff,sizeof(long long)*ncontig,cudaMemcpyHostToDevice,st));
    CUDA_TRY(cudaMemcpyAsync(g->d_clen,clen,sizeof(long long)*ncontig,cudaMemcpyHostToDevice,st));
    CUDA_TRY(cudaMemcpyAsync(g->d_woff,g->woff.data(),sizeof(long long)*(ncontig+1),cudaMemcpyHostToDevice,st));
    CUDA_TRY(cudaMemcpyAsync(g->d_crank,g->crank.data(),sizeof(int)*ncontig,cudaMemcpyHostToDevice,st));
    CUDA_TRY(cudaMemcpyAsync(g->d_perm,g->perm.data(),sizeof(int)*ncontig,cudaMemcpyHostToDevice,st));
  }
  g->h2d_bytes = bps_bytes + (long long) ncontig*(3*8+2*4) + 8;
  int rc;
  { stage_timer t(&g_timings.stage_ms,st);
    rc = fgb_stage_genome_device(d_bps,d_boff,g->d_clen,g->d_woff,ncontig,w,g->d_seq,g->d_rseq,st);
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  if (rc) return rc;
  *out = g.release();
  return FGB_OK;
}

extern "C" void fgb_genome_free(fgb_genome *g) { delete g; }

extern "C" int fgb_genome_perm(const fgb_genome *g, int *perm_out)
{ memcpy(perm_out,g->perm.data(),sizeof(int)*g->ncontig); return FGB_OK; }

//  staged words back to the host (tests): seq (rev=0) or its reverse complement (rev=1)
extern "C" int fgb_genome_download(const fgb_genome *g, int rev, unsigned long long *words,
                                   long long *woff_out)
{ const u64 *src = rev ? g->d_rseq : g->d_seq;
  if (src == NULL) return FGB_ERR_ARG;
  CUDA_TRY(cudaMemcpy(words,src,sizeof(u64)*g->total_words,cudaMemcpyDeviceToHost));
  memcpy(woff_out,g->woff.data(),sizeof(long long)*(g->ncontig+1));
  return FGB_OK;
}
extern "C" long long fgb_genome_words(const fgb_genome *g) { return g->total_words; }

/***********************************************************************************************
 *  GIX
 **********************************************************************************************/

extern "C" void fgb_gix_free(fgb_gix *x) { delete x; }

static void gix_bytes(const fgb_genome *g, fgb_gix *x)        // GIXmake.c:1888-1901
{ long long cum;
  x->post_bytes = 0;
  for (cum = 1; cum < g->maxlen; cum *= 256) x->post_bytes += 1;
  x->cont_bytes = 0;
  for (cum = 1; cum < 2ll*g->ncontig; cum *= 256) x->cont_bytes += 1;
}

//  K1..K4: syncmer scan -> 128-bit records laid out by prefix bin -> bucket sort on the whole record ->
//  2^24 prefix index.

#define GIX_FWD_ONLY 0x80000000u     // flag bit carried in `phi` down to the syncmer scan

//  How the syncmer scan laid its records out for the k-mer sort (fgb_kmer_sort_device): in runs by the first
//  digit of the k-mer partition, bits [fsh, fsh+dbits) of the 12-base prefix, with the histogram of the 8
//  prefix bits above it in hist.  dbits = 0: no layout, the records are in any order.
struct scan_layout
{ int fsh = 0, dbits = 0;
  dblock<unsigned long long> hist;
};

//  Words a table build reads back from the device, in pinned memory so that their copies do not wait: the count
//  pass's record total, the reverse entries it left out, the sampler histogram and the k-mer sort plan's counters.
struct gix_words
{ u64 total, buck[1024], rdropped;                    // buck and rdropped: the count pass's 1025 words
  unsigned plan[4];
};

//  One table build.  The host waits only where it needs a count from the device: once after the count pass (the
//  record total sizes the record block and the sort) and once at the end (the plan's count of bins too large for
//  the bucket sort; there are none in the normal case).  Every block the queued work reads, on the host or the
//  device, lives here until the wait after it.  The builds of a pair run each step on both tables before the
//  wait, so a pair waits twice.
struct gix_job
{ const fgb_genome *g = nullptr;
  unsigned plo = 0, phi = 0, flags = 0;
  bool index = true;
  std::unique_ptr<fgb_gix> x;
  scan_layout lay;
  std::vector<int> tc, ts;
  int ntiles = 0;
  dblock<int> d_tc, d_ts; dblock<unsigned> d_cnt;
  dblock<u64> d_buck, d_total; dblock<unsigned char> d_tmp;
  dblock<rec128> d_a, d_b; dblock<unsigned char> d_stmp, d_plan;
  long long n = 0;
  int inb = 0;
  gix_words *hw = nullptr;
};

//  pinned words for the (at most two) builds a thread has in flight, allocated once
static int pinned_words(gix_job &J, int k)
{ static thread_local gix_words *w = nullptr;
  if (w == nullptr) CUDA_TRY(cudaHostAlloc((void **) &w,2*sizeof(gix_words),cudaHostAllocDefault));
  J.hw = w + k;
  return FGB_OK;
}

static int gix_job_init(gix_job &J, const fgb_genome *g, unsigned plo, unsigned phi_flags, bool index, int k)
{ J.g = g; J.plo = plo; J.phi = phi_flags & ~GIX_FWD_ONLY; J.flags = phi_flags; J.index = index;
  J.x.reset(new fgb_gix());
  gix_bytes(g,J.x.get());
  J.x->ncontig = g->ncontig;
  J.x->fwd_only = (phi_flags & GIX_FWD_ONLY) ? 1 : 0;
  return pinned_words(J,k);
}

//  K1, count pass: syncmer records of the contigs selected by `mask` (NULL: all) counted per tile and first digit
//  of the k-mer partition, at the resolution the k-mer sort would pick for an upper bound of n (two records per
//  scanned position); the total, the reverse entries left out (fwd-only) and the sampler histogram go to J.hw.
static int gix_count(gix_job &J, const unsigned char *mask, cudaStream_t st)
{ const fgb_genome *g = J.g;
  int T = fgb_sc_tile();
  long long npos = 0;
  for (int c = 0; c < g->ncontig; c++)
    if (g->clen[c] >= 12 && g->boff[c] >= 0 && (mask == NULL || mask[c]))
      { npos += g->clen[c] - 11;
        for (long long t0 = 0; t0 + 12 <= g->clen[c]; t0 += T)
          { J.tc.push_back(c); J.ts.push_back((int) t0); }
      }
  J.ntiles = (int) J.tc.size();
  scan_layout &lay = J.lay;
  fgb_kmer_first_digit(2*npos,J.plo,J.phi > J.plo ? J.phi : J.plo + 1,&lay.fsh,&lay.dbits);    // an empty range still gets one bin
  const long long ncnt = (long long) J.ntiles << lay.dbits;
  const long long tmpb = fgb_dev_scan_tmp_bytes(ncnt);
  CUDA_TRY(lay.hist.alloc(256,st));
  CUDA_TRY(J.d_tc.alloc(J.ntiles+1,st));
  CUDA_TRY(J.d_ts.alloc(J.ntiles+1,st));
  CUDA_TRY(J.d_cnt.alloc(ncnt+1,st));
  CUDA_TRY(J.d_buck.alloc(1025,st));
  CUDA_TRY(J.d_total.alloc(1,st));
  CUDA_TRY(J.d_tmp.alloc(tmpb,st));
  CUDA_TRY(cudaMemcpyAsync(J.d_tc,J.tc.data(),sizeof(int)*J.ntiles,cudaMemcpyHostToDevice,st));
  CUDA_TRY(cudaMemcpyAsync(J.d_ts,J.ts.data(),sizeof(int)*J.ntiles,cudaMemcpyHostToDevice,st));
  lazy_timer t(&g_timings.scan_ms,st);
  int rc = fgb_syncmer_digit_count_device(g->d_seq,g->d_clen,g->d_woff,g->d_crank,J.d_tc,J.d_ts,J.ntiles,J.d_buck,
                                          J.d_cnt,lay.fsh,lay.dbits,lay.hist,J.d_total,J.d_tmp,tmpb,J.plo,J.flags,st);
  if (rc) return rc;
  CUDA_TRY(cudaMemcpyAsync(&J.hw->total,J.d_total,8,cudaMemcpyDeviceToHost,st));
  CUDA_TRY(cudaMemcpyAsync(J.hw->buck,J.d_buck,8*1025,cudaMemcpyDeviceToHost,st));
  return FGB_OK;
}

//  K2, emit pass (after the wait for the total): the J.n records into J.d_a (room for n+1), in runs by the first
//  digit of the partition.
static int gix_emit(gix_job &J, cudaStream_t st)
{ if (J.hw->total >= 0xfffffff0ull) return FGB_ERR_LIMIT;
  J.n = (long long) J.hw->total;
  CUDA_TRY(J.d_a.alloc(J.n+1,st));
  lazy_timer t(&g_timings.scan_ms,st);
  return fgb_syncmer_digit_emit_device(J.g->d_seq,J.g->d_clen,J.g->d_woff,J.g->d_crank,J.d_tc,J.d_ts,J.ntiles,
                                       J.d_cnt,J.lay.fsh,J.lay.dbits,J.n,J.d_a,J.plo,J.flags,st);
}

//  K3/K4: sorts the J.n records in J.d_a whose 12-base prefixes lie in [plo,phi), laid out as lay says, and builds
//  the prefix index and the LCP bytes; the plan's counters go to J.hw.
static int gix_sort(gix_job &J, const scan_layout &lay, cudaStream_t st)
{ fgb_gix *x = J.x.get();
  const long long n = J.n, stmpb = fgb_sort128_tmp_bytes(n), planb = fgb_kmer_plan_bytes(n,J.plo,J.phi,lay.fsh,lay.dbits);
  int rc;
  x->n = n;
  CUDA_TRY(J.d_b.alloc(n+1,st));
  CUDA_TRY(J.d_stmp.alloc(stmpb,st));
  CUDA_TRY(J.d_plan.alloc(planb,st));
  if (J.index)
    { CUDA_TRY(x->d_pstart.alloc((1<<24)+1+8,st));
      CUDA_TRY(x->d_adj.alloc((size_t) n + 32,st));
    }
  { lazy_timer t(&g_timings.ksort_ms,st);
    rc = fgb_kmer_sort_device(J.d_a,J.d_b,n,J.plo,J.phi,lay.fsh,lay.dbits,lay.hist,J.d_stmp,stmpb,J.d_plan,&J.inb,st);
  }
  if (rc) return rc;
  CUDA_TRY(cudaMemcpyAsync(J.hw->plan,J.d_plan,16,cudaMemcpyDeviceToHost,st));
  if (J.index)
    { lazy_timer t(&g_timings.index_ms,st);
      rc = fgb_kix_index_device(J.inb ? J.d_b : J.d_a,n,x->d_pstart,x->d_adj,st);
    }
  return rc;
}

//  After the last wait: the bins too large for the bucket sort, if the plan found any (then the index is built
//  again over the finished table), and the handle.
static int gix_done(gix_job &J, cudaStream_t st, fgb_gix **out)
{ fgb_gix *x = J.x.get();
  dblock<rec128> &tab = J.inb ? J.d_b : J.d_a;
  int rc;
  if (J.hw->plan[1] > 0)
    { { lazy_timer t(&g_timings.ksort_ms,st);
        rc = fgb_kmer_sort_oversized(J.inb ? J.d_a : J.d_b,tab,J.n,J.d_plan,J.hw->plan[1],J.hw->plan[2],st);
      }
      if (rc) return rc;
      if (J.index)
        { lazy_timer t(&g_timings.index_ms,st);
          if ((rc = fgb_kix_index_device(tab,J.n,x->d_pstart,x->d_adj,st))) return rc;
        }
    }
  x->d_tab = std::move(tab);
  memcpy(x->buck1024,J.hw->buck,8*1024);
  x->n_both = J.n + (long long) J.hw->rdropped;
  *out = J.x.release();
  return FGB_OK;
}

//  FGB_KSORT_PARTITION=1: the sort ignores the scan's layout and runs every partition pass in Onesweep, a
//  second, independent route to the same table (both can be compared in one process)
static const scan_layout &sort_layout(const gix_job &J)
{ static const scan_layout none;
  const char *part_env = getenv("FGB_KSORT_PARTITION");
  return (part_env != NULL && atoi(part_env) != 0) ? none : J.lay;
}

//  The tables of njob genomes, each step queued for all of them before the wait that follows it: two host waits
//  for the lot.  Only a table with bins too large for the bucket sort waits more, and then its index is queued
//  again after the last wait.
static int gix_build_jobs(gix_job *J, int njob, fgb_gix **out, cudaStream_t st)
{ int rc;
  for (int k = 0; k < njob; k++)
    if ((rc = gix_count(J[k],NULL,st))) return rc;
  CUDA_TRY(fgb_stream_wait(st));
  for (int k = 0; k < njob; k++)
    if ((rc = gix_emit(J[k],st)) || (rc = gix_sort(J[k],sort_layout(J[k]),st))) return rc;
  CUDA_TRY(fgb_stream_wait(st));
  for (int k = 0; k < njob; k++)
    if ((rc = gix_done(J[k],st,out + k))) return rc;
  return FGB_OK;
}

//  index = false: the table only, without prefix index and LCP bytes (the T1 side of a merge reads neither).
//  Returns when the table is complete.
static int gix_build_range(const fgb_genome *g, unsigned plo, unsigned phi_flags, bool index, fgb_gix **out,
                           void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  gix_job J;
  int rc = gix_job_init(J,g,plo,phi_flags,index,0);
  if (!rc) rc = gix_build_jobs(&J,1,out,st);
  if (rc) return rc;
  if (J.hw->plan[1] != 0) CUDA_TRY(fgb_stream_wait(st));        // the index built again after the oversized bins
  return FGB_OK;
}

extern "C" int fgb_gix_build(const fgb_genome *g, fgb_gix **out, void *stream)
{ return gix_build_range(g,0u,1u << 24,true,out,stream); }

//  Forward-strand entries only: the table of the genome that supplies the adaptamers.  Reverse
//  entries of T1 never seed (FastGA.c:921-928), so the fused path does not build, sort or read them.
extern "C" int fgb_gix_build_forward(const fgb_genome *g, fgb_gix **out, void *stream)
{ return gix_build_range(g,0u,(1u << 24) | GIX_FWD_ONLY,true,out,stream); }

//  Only the k-mers whose 12-base prefix lies in [plo,phi): one prefix range of a table, binned and
//  sorted relative to plo.
extern "C" int fgb_gix_build_range(const fgb_genome *g, unsigned plo, unsigned phi, fgb_gix **out, void *stream)
{ if (plo > phi || phi > (1u << 24)) return FGB_ERR_ARG;
  return gix_build_range(g,plo,phi,true,out,stream);
}

/***********************************************************************************************
 *  Building blocks of the k-mer-space sharded path (several GPUs, fastga_b200/shard.py): every rank
 *  scans ITS contigs of both genomes, the k-mer records travel to the rank that owns their prefix
 *  range, each rank merges its slice of the two tables, and the seeds travel to the rank that owns
 *  their A-contig.  Nothing is replicated; the two exchanges are all-to-alls of 16-byte records.
 **********************************************************************************************/

//  unsorted k-mer records of the contigs with mask[c] != 0 (device buffer handed to the caller:
//  fgb_device_free); fwd_only: forward-strand entries only (the adaptamer side).  The scan's layout is
//  dropped: the caller regroups the records by owner and each owner sorts its share from any order.
extern "C" int fgb_kmers_scan(const fgb_genome *g, const unsigned char *mask, int fwd_only,
                              void **d_recs, long long *n, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  gix_job J;
  int rc = gix_job_init(J,g,0u,(1u << 24) | (fwd_only ? GIX_FWD_ONLY : 0u),false,0);
  if (!rc) rc = gix_count(J,mask,st);
  if (rc) return rc;
  CUDA_TRY(fgb_stream_wait(st));
  if ((rc = gix_emit(J,st))) return rc;
  CUDA_TRY(fgb_stream_wait(st));                        // the records are the caller's from here on
  *n = J.n;
  *d_recs = J.d_a.release();
  return FGB_OK;
}

//  a table over n unsorted device records (copied) whose 12-base prefixes lie in [plo,phi): one
//  rank's slice of a k-mer-space sharded table.  The range is a precondition this call does not check: a
//  record outside it wraps the fine-bin and sub-bin arithmetic of fgb_kmer_sort_device, so it is dropped
//  silently or sends kmer_bucket_sort_kernel's cnt[] index out of bounds.  Refusing such records would need a
//  device check before the bucket sort, and another host wait on the sharded path.
extern "C" int fgb_gix_from_records(const void *d_recs, long long n, unsigned plo, unsigned phi, int fwd_only,
                                    int post_bytes, int cont_bytes, int ncontig, fgb_gix **out, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (n < 0 || n >= 0xfffffff0ll || plo >= phi || phi > (1u << 24)) return FGB_ERR_ARG;
  gix_job J;
  J.plo = plo; J.phi = phi;
  J.x.reset(new fgb_gix());
  J.x->post_bytes = post_bytes; J.x->cont_bytes = cont_bytes; J.x->ncontig = ncontig;
  J.x->fwd_only = fwd_only ? 1 : 0;
  int rc = pinned_words(J,0);
  if (rc) return rc;
  J.hw->rdropped = 0;
  memset(J.hw->buck,0,8*1024);
  J.n = n;
  CUDA_TRY(J.d_a.alloc(n+1,st));
  if (n > 0) CUDA_TRY(cudaMemcpyAsync(J.d_a,d_recs,sizeof(rec128)*n,cudaMemcpyDeviceToDevice,st));
  if ((rc = gix_sort(J,scan_layout(),st))) return rc;
  CUDA_TRY(fgb_stream_wait(st));
  if ((rc = gix_done(J,st,out))) return rc;
  if (J.hw->plan[1] != 0) CUDA_TRY(fgb_stream_wait(st));        // the index built again after the oversized bins
  return FGB_OK;
}

extern "C" long long fgb_gix_size(const fgb_gix *x) { return x->n; }
extern "C" int fgb_gix_post_bytes(const fgb_gix *x) { return x->post_bytes; }
extern "C" int fgb_gix_cont_bytes(const fgb_gix *x) { return x->cont_bytes; }

extern "C" int fgb_gix_download(const fgb_gix *x, void *tab /* n x 16 B */, unsigned *pstart /* 2^24+1 */,
                                unsigned long long *buck1024)
{ if (tab) CUDA_TRY(cudaMemcpy(tab,x->d_tab,sizeof(rec128)*x->n,cudaMemcpyDeviceToHost));
  if (pstart) CUDA_TRY(cudaMemcpy(pstart,x->d_pstart,sizeof(unsigned)*((1<<24)+1),cudaMemcpyDeviceToHost));
  if (buck1024) memcpy(buck1024,x->buck1024,8*1024);
  return FGB_OK;
}

//  A GIX from host-side device-layout records (sorted) -- used to feed tables from elsewhere.
extern "C" int fgb_gix_upload(const void *tab, long long n, int post_bytes, int cont_bytes,
                              int ncontig, fgb_gix **out, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (n >= 0xfffffff0ll) return FGB_ERR_LIMIT;
  std::unique_ptr<fgb_gix> x(new fgb_gix());
  x->n = n; x->n_both = n; x->post_bytes = post_bytes; x->cont_bytes = cont_bytes; x->ncontig = ncontig;
  CUDA_TRY(x->d_tab.alloc(n+1,st));
  CUDA_TRY(x->d_pstart.alloc((1<<24)+1+8,st));
  CUDA_TRY(x->d_adj.alloc((size_t) x->n + 32,st));
  CUDA_TRY(cudaMemcpyAsync(x->d_tab,tab,sizeof(rec128)*n,cudaMemcpyHostToDevice,st));
  int rc = fgb_kix_index_device(x->d_tab,n,x->d_pstart,x->d_adj,st);
  CUDA_TRY(cudaStreamSynchronize(st));
  if (rc) return rc;
  *out = x.release();
  return FGB_OK;
}

//  A GIX from the reference's on-disk form: concatenated .ktab entries (all parts, in order) and
//  the stub's cumulative 2^24 index (libfastk.c:815-840).
extern "C" int fgb_gix_import_ktab(const unsigned char *entries, long long n, int post_bytes,
                                   int cont_bytes, const long long *index, int ncontig,
                                   fgb_gix **out, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (n >= 0xfffffff0ll || post_bytes > 4 || cont_bytes > 2) return FGB_ERR_LIMIT;
  std::unique_ptr<fgb_gix> x(new fgb_gix());
  x->n = n; x->n_both = n; x->post_bytes = post_bytes; x->cont_bytes = cont_bytes; x->ncontig = ncontig;
  long long E = 9 + post_bytes + cont_bytes;
  dblock<unsigned char> d_ent; dblock<long long> d_index;
  CUDA_TRY(d_ent.alloc(E*n + 16,st));
  CUDA_TRY(d_index.alloc(1ll << 24,st));
  CUDA_TRY(x->d_tab.alloc(n+1,st));
  CUDA_TRY(x->d_pstart.alloc((1<<24)+1+8,st));
  CUDA_TRY(x->d_adj.alloc((size_t) x->n + 32,st));
  CUDA_TRY(cudaMemcpyAsync(d_ent,entries,E*n,cudaMemcpyHostToDevice,st));
  CUDA_TRY(cudaMemcpyAsync(d_index,index,8ll<<24,cudaMemcpyHostToDevice,st));
  int rc = fgb_ktab_import_device(d_ent,n,post_bytes,cont_bytes,d_index,x->d_tab,st);
  if (!rc) rc = fgb_kix_index_device(x->d_tab,n,x->d_pstart,x->d_adj,st);
  CUDA_TRY(cudaStreamSynchronize(st));
  if (rc) return rc;
  *out = x.release();
  return FGB_OK;
}

//  On-disk entries for the whole table (host buffer of n*(9+pb+cb) bytes); part_first = entry
//  index at which each .ktab part starts (its LCP byte is 0, MSDsort.c:485-488).
extern "C" int fgb_gix_export_ktab(const fgb_gix *x, const long long *part_first, int nparts,
                                   unsigned char *out, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  long long E = 9 + x->post_bytes + x->cont_bytes;
  dblock<unsigned char> d_out; dblock<long long> d_pf;
  CUDA_TRY(d_out.alloc(E*x->n + 16,st));
  CUDA_TRY(d_pf.alloc(nparts+1,st));
  CUDA_TRY(cudaMemcpyAsync(d_pf,part_first,8*nparts,cudaMemcpyHostToDevice,st));
  int rc = fgb_ktab_export_device(x->d_tab,x->n,x->post_bytes,x->cont_bytes,d_pf,nparts,d_out,st);
  if (!rc) CUDA_TRY(cudaMemcpyAsync(out,d_out,E*x->n,cudaMemcpyDeviceToHost,st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return rc;
}

/***********************************************************************************************
 *  Seeds: adaptamer merge + seed sort
 **********************************************************************************************/

static int bitlen(long long v) { int b = 0; while (v > 0) { b += 1; v >>= 1; } return b; }

extern "C" void fgb_seeds_free(fgb_seeds *s) { delete s; }

static int seeds_find_impl(const fgb_gix *x1, const fgb_gix *x2, long long amxpos,
                           long long bmxpos, int freq, bool self, fgb_seeds **out, void *stream);

extern "C" int fgb_seeds_find(const fgb_gix *x1, const fgb_gix *x2, long long amxpos,
                              long long bmxpos, int freq, fgb_seeds **out, void *stream)
{ return seeds_find_impl(x1,x2,amxpos,bmxpos,freq,false,out,stream); }

//  SELF mode (FastGA A): the table against itself (new_self_merge_thread, FastGA.c:1616)
extern "C" int fgb_seeds_find_self(const fgb_gix *x, long long amxpos, int freq, fgb_seeds **out, void *stream)
{ return seeds_find_impl(x,x,amxpos,amxpos,freq,true,out,stream); }

struct seed_bits { int anti, band, jc, ic, key; };

static int seed_layout_of(const fgb_gix *x1, const fgb_gix *x2, long long amxpos, long long bmxpos, seed_bits *L)
{ L->anti = bitlen(amxpos + bmxpos);
  L->band = L->anti > 6 ? L->anti - 6 : 1;
  L->jc   = bitlen(x2->ncontig > 1 ? x2->ncontig-1 : 1);
  L->ic   = bitlen(x1->ncontig > 1 ? x1->ncontig-1 : 1);
  L->key  = 12 + L->anti + L->band + L->jc + L->ic + 1;
  return L->key > 128 ? FGB_ERR_LIMIT : FGB_OK;
}

//  K5: the unsorted seed records of x1 against x2 in a fresh device buffer (room for n+1)
static int seeds_merge_impl(const fgb_gix *x1, const fgb_gix *x2, long long amxpos, long long bmxpos, int freq,
                            bool self, const seed_bits &L, dblock<rec128> &d_out, long long *nseeds_out,
                            long long *sumlen_out, long long *n1m_out, cudaStream_t st)
{ if (self && x1->fwd_only) return FGB_ERR_ARG;                // SELF mode needs both strands
  dblock<u64> d_counters; dblock<rec128> d_fwd, d_a;
  int rc;
  u64 nseeds = 0, sumlen = 0;
  //  the adaptamer side must be a forward-strand table (reverse entries never seed): a both-strand
  //  table (imported .ktab, fgb_gix_build) is compacted once; the fused path builds it forward-only
  const rec128 *t1 = x1->d_tab; long long n1 = x1->n;
  CUDA_TRY(d_counters.alloc(2,st));
  if (!self && !x1->fwd_only && n1 > 0)
    { CUDA_TRY(d_fwd.alloc(n1+1,st));
      if ((rc = fgb_forward_view_device(x1->d_tab,n1,d_fwd,&n1,st))) return rc;
      t1 = d_fwd;
    }
  long long cap = (self ? 2*x1->n : 2*n1 + (n1 >> 1)) + 1024;
  for (int attempt = 0; ; attempt++)
    { CUDA_TRY(d_a.alloc(cap+1,st));
      if (self)
        rc = fgb_self_merge_device(x1->d_tab,x1->n,x1->d_pstart,freq,L.anti,L.band,L.jc,L.ic,amxpos,
                                   d_a,cap,d_counters,&nseeds,&sumlen,st);
      else
        rc = fgb_merge_device(t1,n1,x2->d_tab,x2->n,x2->d_pstart,x2->d_adj,freq,L.anti,L.band,L.jc,L.ic,
                              amxpos,bmxpos,d_a,cap,d_counters,&nseeds,&sumlen,st);
      if (rc == FGB_OK) break;
      d_a.reset();                                              // before the larger buffer is allocated
      if (rc != FGB_ERR_OVERFLOW || attempt > 0) return rc;
      cap = (long long) nseeds + 1024;
      g_timings.merge_ms = 0; g_timings.merge_launches = 0;   // only the successful launch is reported
    }
  if (nseeds >= 0xfffffff0ull) return FGB_ERR_LIMIT;
  d_out = std::move(d_a); *nseeds_out = (long long) nseeds; *sumlen_out = (long long) sumlen; *n1m_out = n1;
  return FGB_OK;
}

//  First key bit of the seed sort.  The lcp field (bits 0..5) never breaks a tie: two seeds that agree on
//  strand, contigs, band, anti-diagonal and diagonal remainder are the same pair of positions.  Records
//  that make_seed built in the same call (the merges of merge.cu) skip bit 6 too: forward seeds have
//  diag = bmxpos + (i - j) and anti = i + j, complement seeds diag = maxdag - (i + j) and
//  anti = amxpos - (i - j), so on either strand diag & 1 (bit 6) is anti & 1 (bit 12) XOR a constant of
//  the strand (the key's top bit).  Both are sorted above bit 6, so [7, key) gives the order of
//  [6, key) -- one 8-bit pass less on a key of 57 to 64 bits.  Records from a caller
//  (fgb_seeds_from_records) keep bit 6.
#define SEED_SORT_LO_ANY    6
#define SEED_SORT_LO_MERGED 7

//  K6: sorts n seed records in d_a (consumed) into a handle, on key bits [bit_lo, L.key)
static int seeds_sort_impl(dblock<rec128> d_a, long long n, const seed_bits &L, int bit_lo, long long amxpos,
                           long long bmxpos, bool self, long long sumlen, long long n1m, fgb_seeds **out,
                           cudaStream_t st)
{ dblock<rec128> d_b; dblock<unsigned char> d_tmp;
  std::unique_ptr<fgb_seeds> s(new fgb_seeds());
  s->self_mode = self ? 1 : 0;
  s->anti_bits = L.anti; s->band_bits = L.band; s->jc_bits = L.jc; s->ic_bits = L.ic;
  s->amxpos = amxpos; s->bmxpos = bmxpos;
  s->n = n; s->sumlen = sumlen; s->n1_merged = n1m;
  long long tmpb = fgb_sort128_tmp_bytes(n);
  int rc, inb = 0;
  //  a key of <= 64 bits leaves hi = 0 in every record: the passes run on the lo words alone.
  //  FGB_SEED_SORT_WIDE=1 forces the 128-bit passes (both paths can be compared in one process).
  const char *wide_env = getenv("FGB_SEED_SORT_WIDE");
  const bool narrow = L.key <= 64 && !(wide_env != NULL && atoi(wide_env) != 0);
  u64 hiflag = 0, *d_hiflag = NULL;
  CUDA_TRY(d_b.alloc(n+1,st));
  CUDA_TRY(d_tmp.alloc(tmpb,st));
  { stage_timer t(&g_timings.ssort_ms,st);
    rc = fgb_radix_sort_device(d_a,d_b,n,bit_lo,L.key,narrow,d_tmp,tmpb,&inb,&d_hiflag,st);
  }
  if (rc) return rc;
  if (d_hiflag) CUDA_TRY(cudaMemcpyAsync(&hiflag,d_hiflag,8,cudaMemcpyDeviceToHost,st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (hiflag) return FGB_ERR_ARG;                      // a record with hi != 0: the 64-bit passes mis-ordered it
  s->d_rec = std::move(inb ? d_b : d_a);
  *out = s.release();
  return FGB_OK;
}

static int seeds_find_impl(const fgb_gix *x1, const fgb_gix *x2, long long amxpos,
                           long long bmxpos, int freq, bool self, fgb_seeds **out, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  seed_bits L;
  int rc = seed_layout_of(x1,x2,amxpos,bmxpos,&L);
  if (rc) return rc;
  dblock<rec128> d_a; long long n = 0, sumlen = 0, n1m = 0;
  if ((rc = seeds_merge_impl(x1,x2,amxpos,bmxpos,freq,self,L,d_a,&n,&sumlen,&n1m,st))) return rc;
  return seeds_sort_impl(std::move(d_a),n,L,SEED_SORT_LO_MERGED,amxpos,bmxpos,self,sumlen,n1m,out,st);
}

//  ---- sharded path: seeds leave the merge unsorted, travel to their A-contig's owner, are sorted there ----

//  unsorted seed records of x1 against x2 (device buffer handed to the caller: fgb_device_free);
//  bits[4] = anti, band, jcont, icont field widths; info[2] = sum of seed lengths, T1 entries merged
extern "C" int fgb_seeds_merge(const fgb_gix *x1, const fgb_gix *x2, long long amxpos, long long bmxpos, int freq,
                               void **d_seeds, long long *n, int *bits, long long *info, void *stream)
{ seed_bits L;
  int rc = seed_layout_of(x1,x2,amxpos,bmxpos,&L);
  if (rc) return rc;
  dblock<rec128> d_a; long long sumlen = 0, n1m = 0;
  if ((rc = seeds_merge_impl(x1,x2,amxpos,bmxpos,freq,false,L,d_a,n,&sumlen,&n1m,(cudaStream_t) stream))) return rc;
  *d_seeds = d_a.release();
  bits[0] = L.anti; bits[1] = L.band; bits[2] = L.jc; bits[3] = L.ic;
  if (info) { info[0] = sumlen; info[1] = n1m; }
  return FGB_OK;
}

//  Count + scatter of n 16-byte records by owner[field], field = the nbits bits at bit pos of the record
//  (nowner entries): d_out[bounds[w] .. bounds[w+1]) are the records of owner w, order inside a group free.
//  Every owner entry must name a rank of the world: the kernel indexes its per-rank counters with it.
static int group_by_owner(const void *d_src, long long n, int pos, int nbits, const int *owner, int nowner,
                          int world, void *d_out, long long *bounds, cudaStream_t st)
{ if (world < 1 || world > 64) return FGB_ERR_ARG;
  for (int i = 0; i < nowner; i++)
    if (owner[i] < 0 || owner[i] >= world) return FGB_ERR_ARG;
  for (int w = 0; w <= world; w++) bounds[w] = 0;
  if (n <= 0) return FGB_OK;
  dblock<int> d_owner; dblock<u64> d_cnt;
  int rc;
  u64 cnt[64], base[65];
  CUDA_TRY(d_owner.alloc((size_t) nowner,st));
  CUDA_TRY(d_cnt.alloc(64*2,st));
  CUDA_TRY(cudaMemcpyAsync(d_owner,owner,sizeof(int)*(size_t) nowner,cudaMemcpyHostToDevice,st));
  CUDA_TRY(cudaMemsetAsync(d_cnt,0,8*64*2,st));
  if ((rc = fgb_owner_count_device(d_src,n,pos,nbits,d_owner,nowner,world,d_cnt,st))) return rc;
  CUDA_TRY(cudaMemcpyAsync(cnt,d_cnt,8*64,cudaMemcpyDeviceToHost,st));
  CUDA_TRY(cudaStreamSynchronize(st));
  base[0] = 0;
  for (int w = 0; w < world; w++) base[w+1] = base[w] + cnt[w];
  CUDA_TRY(cudaMemcpyAsync(d_cnt + 64,base,8*64,cudaMemcpyHostToDevice,st));
  if ((rc = fgb_owner_scatter_device(d_src,n,pos,nbits,d_owner,nowner,world,d_cnt + 64,d_out,st))) return rc;
  CUDA_TRY(cudaStreamSynchronize(st));
  for (int w = 0; w <= world; w++) bounds[w] = (long long) base[w];
  return FGB_OK;
}

//  seeds grouped by the rank that owns their A-contig: owner[r] for contig RANK r (the icont field)
extern "C" int fgb_seeds_group_by_owner(const void *d_seeds, long long n, const int *bits, const int *owner,
                                        int nrank_contigs, int world, void *d_out, long long *bounds,
                                        void *stream)
{ return group_by_owner(d_seeds,n,12 + bits[0] + bits[1] + bits[2],bits[3],owner,nrank_contigs,world,d_out,bounds,
                        (cudaStream_t) stream);
}

//  k-mer records grouped by the rank that owns their first four bases: owner256[b] for top byte b
extern "C" int fgb_records_group_by_owner(const void *d_recs, long long n, const int *owner256, int world,
                                          void *d_out, long long *bounds, void *stream)
{ return group_by_owner(d_recs,n,120,8,owner256,256,world,d_out,bounds,(cudaStream_t) stream); }

//  sorted seed set over n unsorted device records (copied); bits as fgb_seeds_merge returns them
extern "C" int fgb_seeds_from_records(const void *d_recs, long long n, const int *bits, long long amxpos,
                                      long long bmxpos, long long sumlen, fgb_seeds **out, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (n < 0 || n >= 0xfffffff0ll) return FGB_ERR_LIMIT;
  seed_bits L;
  L.anti = bits[0]; L.band = bits[1]; L.jc = bits[2]; L.ic = bits[3];
  L.key = 12 + L.anti + L.band + L.jc + L.ic + 1;
  if (L.key > 128) return FGB_ERR_LIMIT;
  dblock<rec128> d_a;
  CUDA_TRY(d_a.alloc(n+1,st));
  if (n > 0) CUDA_TRY(cudaMemcpyAsync(d_a,d_recs,sizeof(rec128)*n,cudaMemcpyDeviceToDevice,st));
  return seeds_sort_impl(std::move(d_a),n,L,SEED_SORT_LO_ANY,amxpos,bmxpos,false,sumlen,0,out,st);
}

extern "C" long long fgb_seeds_size(const fgb_seeds *s) { return s->n; }
extern "C" long long fgb_seeds_sumlen(const fgb_seeds *s) { return s->sumlen; }
extern "C" int fgb_seeds_layout(const fgb_seeds *s, int *bits /* anti, band, jc, ic */)
{ bits[0] = s->anti_bits; bits[1] = s->band_bits; bits[2] = s->jc_bits; bits[3] = s->ic_bits; return FGB_OK; }
extern "C" int fgb_seeds_download(const fgb_seeds *s, void *rec)
{ CUDA_TRY(cudaMemcpy(rec,s->d_rec,sizeof(rec128)*s->n,cudaMemcpyDeviceToHost)); return FGB_OK; }

//  Plain host-buffer sort of 16-byte records on key bytes [byte_lo,byte_hi): the building block
//  behind both drop-in sort seams.
extern "C" int fgb_sort128_host(void *recs, long long n, int byte_lo, int byte_hi, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  dblock<rec128> d_a, d_b; dblock<unsigned char> d_tmp;
  long long tmpb = fgb_sort128_tmp_bytes(n);
  CUDA_TRY(d_a.alloc(n+1,st));
  CUDA_TRY(d_b.alloc(n+1,st));
  CUDA_TRY(d_tmp.alloc(tmpb,st));
  CUDA_TRY(cudaMemcpyAsync(d_a,recs,sizeof(rec128)*n,cudaMemcpyHostToDevice,st));
  int inb = 0;
  int rc = fgb_sort128_device(d_a,d_b,n,byte_lo,byte_hi,d_tmp,tmpb,&inb,st);
  if (!rc) CUDA_TRY(cudaMemcpyAsync(recs,inb ? d_b : d_a,sizeof(rec128)*n,cudaMemcpyDeviceToHost,st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return rc;
}

extern "C" int fgb_device_ready()
{ int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return 0;
  return 1;
}

/***********************************************************************************************
 *  Whole path, host buffers in / host records out: what `FastGA -1:<out> A B` computes between
 *  Read_GDB and la_merge (FastGA.c:4927-5205), GIX construction included.
 **********************************************************************************************/

//  The whole path on staged genomes: k-mer tables -> adaptamer merge -> seed sort -> extension -> filter.
//  self: SELF mode (`FastGA A`, B == A): one both-strand table merged against itself by the self block
//  rule, and the band borders of align_contigs for a contig against itself.
static int align_pipeline(const fgb_genome *A, const fgb_genome *B, bool self, const float *freqA, int freq,
                          int chain_break, int chain_min, int align_min, double align_rate, fgb_alns **out,
                          fgb_run_stats *stats, cudaStream_t st)
{ fgb_run_stats s = {};
  fgb_seeds *ps = NULL; fgb_overlaps *po = NULL;
  int rc;
  long long t0 = now_us(), t1, t2, t3, t4;
  { std::unique_ptr<fgb_gix> x1, x2;
    fgb_gix *p[2] = { NULL, NULL };
    const long long w0 = g_waits;
    { gix_job J[2];
      //  pair: the adaptamer side forward strand only, and only the table (the merge reads B's index)
      rc = gix_job_init(J[0],A,0u,(1u << 24) | (self ? 0u : GIX_FWD_ONLY),self,0);
      if (!rc && !self) rc = gix_job_init(J[1],B,0u,1u << 24,true,1);
      if (!rc) rc = gix_build_jobs(J,self ? 1 : 2,p,st);
      x1.reset(p[0]); x2.reset(p[1]);
      if (rc) return rc;
    }
    s.gix_waits = g_waits - w0;
    const fgb_gix *xb = self ? x1.get() : x2.get();
    t1 = now_us();
    s.nkmers1 = x1->n_both; s.nkmers2 = xb->n;
    seed_bits L;
    dblock<rec128> d_a; long long n = 0;
    rc = seed_layout_of(x1.get(),xb,A->maxlen,B->maxlen,&L);
    if (!rc) rc = seeds_merge_impl(x1.get(),xb,A->maxlen,B->maxlen,freq,self,L,d_a,&n,&s.sumlen,&s.nkmers1_fwd,st);
    //  the tables go back to the allocator as soon as the merge has read them (two tables + seeds + sort
    //  buffer of a multi-Gbp pair do not fit side by side)
    x1.reset(); x2.reset();
    if (!rc) rc = seeds_sort_impl(std::move(d_a),n,L,SEED_SORT_LO_MERGED,A->maxlen,B->maxlen,self,s.sumlen,
                                  s.nkmers1_fwd,&ps,st);
  }
  if (rc) return rc;
  std::unique_ptr<fgb_seeds> sd(ps);
  s.nseeds = sd->n;
  t2 = now_us();
  std::vector<short> tables(65536);
  int ave = 0;
  fgb_align_spec(1.-align_rate,freqA,tables.data(),&ave);           // FastGA.c:3760
  rc = fgb_extend(sd.get(),A,B,chain_break,chain_min,align_min,align_rate,tables.data(),ave,100,&po,st);
  t3 = now_us();
  const int jb = sd->jc_bits, ib = sd->ic_bits;
  sd.reset();
  if (rc) return rc;
  std::unique_ptr<fgb_overlaps> ov(po);
  rc = fgb_filter(ov.get(),A->perm.data(),B->perm.data(),jb,ib,1,out);
  t4 = now_us();
  const ext_counters &c = ov->counters;
  s.us_gix = t1-t0; s.us_seeds = t2-t1; s.us_extend = t3-t2; s.us_filter = t4-t3;
  s.nhits = (long long) c.hits; s.nla = (long long) c.la_calls; s.nwaves = (long long) c.waves;
  s.ncells = (long long) c.cells; s.nseg = (long long) c.nseg; s.nwork = (long long) c.nwork;
  s.warp_cycles = (long long) c.warp_cycles; s.wave_cycles = (long long) c.wave_cycles;
  s.extract_cycles = (long long) c.extract_cycles;
  s.slow_cycles = (long long) ((c.slowest_warp >> 40) << 12); s.slow_waves = (long long) ((c.slowest_warp >> 16) & 0xffffff);
  s.paired_waves = (long long) c.paired_waves; s.pairings = (long long) c.pairings;
  s.h2d_bytes = A->h2d_bytes + (self ? 0 : B->h2d_bytes) + 65536*2;
  s.d2h_bytes = fgb_overlaps_bytes(ov.get()) + 16 + 8*1024*(self ? 1 : 2) + 64;    // 8 KB of bucket counts per table
  if (stats) *stats = s;
  return rc;
}

//  Device-resident genomes in, final alignments out (the timed "step" of bench.py).
extern "C" int fgb_align_resident(const fgb_genome *A, const fgb_genome *B, const float *freqA,
                                  int freq, int chain_break, int chain_min, int align_min,
                                  double align_rate, fgb_alns **out, fgb_run_stats *stats, void *stream)
{ return align_pipeline(A,B,false,freqA,freq,chain_break,chain_min,align_min,align_rate,out,stats,
                        (cudaStream_t) stream);
}

//  The reference-facing calls: host .bps images + contig tables in, alignments out; every
//  host<->device copy happens inside.
extern "C" int fgb_fastga_self(const unsigned char *bps, long long nb, int nc, const long long *clen,
                               const long long *boff, const float *freq4,
                               int freq, int chain_break, int chain_min, int align_min, double align_rate,
                               fgb_alns **out, fgb_run_stats *stats, void *stream)
{ fgb_genome *p = NULL;
  int rc;
  if ((rc = fgb_genome_create(bps,nb,nc,clen,boff,1,&p,stream))) return rc;
  std::unique_ptr<fgb_genome> A(p);
  return align_pipeline(A.get(),A.get(),true,freq4,freq,chain_break,chain_min,align_min,align_rate,out,stats,
                        (cudaStream_t) stream);
}

extern "C" int fgb_fastga(const unsigned char *bpsA, long long nbA, int ncA, const long long *clenA,
                          const long long *boffA, const float *freqA,
                          const unsigned char *bpsB, long long nbB, int ncB, const long long *clenB,
                          const long long *boffB,
                          int freq, int chain_break, int chain_min, int align_min, double align_rate,
                          fgb_alns **out, fgb_run_stats *stats, void *stream)
{ fgb_genome *p = NULL;
  int rc;
  if ((rc = fgb_genome_create(bpsA,nbA,ncA,clenA,boffA,1,&p,stream))) return rc;
  std::unique_ptr<fgb_genome> A(p);
  if ((rc = fgb_genome_create(bpsB,nbB,ncB,clenB,boffB,0,&p,stream))) return rc;
  std::unique_ptr<fgb_genome> B(p);
  return align_pipeline(A.get(),B.get(),false,freqA,freq,chain_break,chain_min,align_min,align_rate,out,stats,
                        (cudaStream_t) stream);
}
