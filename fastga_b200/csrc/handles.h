// Opaque handle layouts behind the C-ABI (include/fastga_b200.h only forward-declares them).  A handle
// owns its device blocks: fgb_*_free is `delete`.
#pragma once
#include "common.cuh"
#include <memory>
#include <vector>

struct fgb_timings            // device milliseconds per stage (CUDA events on the call's stream)
{ float h2d_ms, stage_ms, scan_ms, ksort_ms, index_ms, merge_ms, ssort_ms, triples_ms, extend_ms,
        d2h_ms, filter_ms;
  int   merge_launches, extend_launches, launches;
};

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

struct fgb_overlaps                        // raw local alignments of fgb_extend, host resident
{ long long nrec = 0, nbytes = 0;
  unsigned char *h_buf = nullptr;          // packed records (OUT_HDR + trace padded to 8), malloc'ed
  unsigned long long counters[16] = {0};
  long long nseg = 0, nwork = 0;
  long long retry[4] = {0};                // fgb_overlaps_retry_info
  fgb_overlaps() = default;
  fgb_overlaps(const fgb_overlaps &) = delete;
  fgb_overlaps &operator=(const fgb_overlaps &) = delete;
  ~fgb_overlaps() { free(h_buf); }
};
