// Opaque handle layouts behind the C-ABI (include/fastga_b200.h only forward-declares them).  A handle
// owns its device blocks: fgb_*_free is `delete`.
#pragma once
#include "../../include/fastga_b200.h"
#include "common.cuh"
#include <stddef.h>
#include <memory>
#include <vector>

struct fgb_genome
{ int ncontig = 0;
  long long seqtot = 0, maxlen = 0, total_words = 0, h2d_bytes = 0;
  std::vector<long long> clen, boff, woff;
  std::vector<int> perm, crank;            // perm[rank] = contig, crank[contig] = rank
  dblock<long long> d_clen, d_woff;
  dblock<int> d_crank, d_perm;
  dblock<unsigned long long> d_seq, d_rseq;
};

struct fgb_gix
{ long long n = 0;
  dblock<rec128> d_tab;
  dblock<unsigned> d_pstart;               // [2^24+1] lower-bound index by 12-base prefix
  dblock<unsigned char> d_adj;             // [n+32] LCP in bases of entries i-1 and i (0 at the table ends)
  unsigned long long buck1024[1024] = {0}; // sampler histogram (decides the .ktab part split)
  int post_bytes = 0, cont_bytes = 0, ncontig = 0;
  int fwd_only = 0;                        // forward-strand entries only (adaptamer side of a merge)
  long long n_both = 0;                    // entries of the both-strand table (= n unless fwd_only)
};

struct fgb_seeds
{ long long n = 0, sumlen = 0;
  dblock<rec128> d_rec;                    // sorted seed records
  int anti_bits = 0, band_bits = 0, jc_bits = 0, ic_bits = 0;
  long long amxpos = 0, bmxpos = 0;
  int self_mode = 0;                       // seeds of a genome against itself (FastGA A)
  long long n1_merged = 0;                 // forward-strand T1 entries the merge consumed
};

//  Header of one raw alignment record of the extension (fgb_overlaps_data); its trace of tlen bytes
//  follows, padded to 8.  launch: the extension launch that emitted it (a re-run triple keeps the
//  records of its last one).
struct ovl_hdr { int triple, seq, pairkey, abpos, bbpos, aepos, bepos, diffs, tlen, launch; };
static_assert(sizeof(ovl_hdr) == 40, "raw record header: 10 ints");

//  bytes of a raw record whose trace is tlen bytes long
static __host__ __device__ __forceinline__ int ovl_bytes(int tlen) { return (int) sizeof(ovl_hdr) + ((tlen + 7) & ~7); }

//  The extension's counters, in the order fgb_overlaps_counters exports them.  extend_kernel adds its
//  warps' counts (or takes their maximum); nseg and nwork are set on the host.  The wait counts are
//  taken in EX_DIAG builds only (0 otherwise).
struct ext_counters
{ unsigned long long hits, la_calls, waves, cells,
                     front_wait,                 // front warps: cycles waiting for ring space
                     nseg, nwork,                // band segments, work triples
                     front_total,                // front warps: waves on the fast path
                     warp_cycles, wave_cycles, extract_cycles,
                     paired_waves,               // waves run by a front/back warp team
                     pairings,                   // passes handed to a team.  EX_DIAG builds: the slowest warp,
                                                 //   cycles >> 12 << 40 | wave cycles >> 12 << 20 | read-out cycles >> 12
                     back_wait,                  // T warps: cycles waiting for their front warp
                     max_warp_cycles,            // the slowest warp's cycles.  EX_DIAG builds: P warps' cycles
                                                 //   waiting for their T warp
                     slowest_warp;               // the slowest warp: cycles >> 12 << 40 | waves << 16 | LA calls
};
static_assert(sizeof(ext_counters) == 16*8, "fgb_overlaps_counters exports 16 counters");
static_assert(offsetof(ext_counters,hits) == 0*8 && offsetof(ext_counters,la_calls) == 1*8 &&
              offsetof(ext_counters,waves) == 2*8 && offsetof(ext_counters,cells) == 3*8 &&
              offsetof(ext_counters,front_wait) == 4*8 && offsetof(ext_counters,nseg) == 5*8 &&
              offsetof(ext_counters,nwork) == 6*8 && offsetof(ext_counters,front_total) == 7*8 &&
              offsetof(ext_counters,warp_cycles) == 8*8 && offsetof(ext_counters,wave_cycles) == 9*8 &&
              offsetof(ext_counters,extract_cycles) == 10*8 && offsetof(ext_counters,paired_waves) == 11*8 &&
              offsetof(ext_counters,pairings) == 12*8 && offsetof(ext_counters,back_wait) == 13*8 &&
              offsetof(ext_counters,max_warp_cycles) == 14*8 && offsetof(ext_counters,slowest_warp) == 15*8,
              "counter export order");

struct fgb_overlaps                        // raw local alignments of fgb_extend, host resident
{ long long nrec = 0, nbytes = 0;
  unsigned char *h_buf = nullptr;          // packed records (ovl_hdr + trace padded to 8), malloc'ed
  ext_counters counters = {};
  long long retry[4] = {0};                // fgb_overlaps_retry_info
  fgb_overlaps() = default;
  fgb_overlaps(const fgb_overlaps &) = delete;
  fgb_overlaps &operator=(const fgb_overlaps &) = delete;
  ~fgb_overlaps() { free(h_buf); }
};
