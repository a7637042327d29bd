// Entry points that one .cu file of the library defines and another calls, beyond the C-ABI of
// include/fastga_b200.h.  The defining file includes this header too, so a definition that drifts
// from its declaration here or in the C-ABI header does not compile.
#pragma once
#include "../../include/fastga_b200.h"
#include "common.cuh"

extern "C" {

// ---- sort128.cu: radix sort of 16-byte records, k-mer table sort ----
//  Stable LSD sort of n records in d_a on the 8-bit digits at bit offsets bit_lo, bit_lo+8, ... below
//  bit_hi (the last digit may reach past bit_hi: the bits above a key are part of the order, zero in
//  every record sorted here); d_b is a scratch of 16(n+1) bytes, d_tmp one of fgb_sort128_tmp_bytes(n).
//  narrow = 0: the result lands in d_a or d_b (*result_in_b).  narrow = 1 (bit_hi <= 64): the records'
//  hi words must be zero, the result lands in d_a, and *d_hiflag points at a device word that gets the
//  OR of every hi word dropped (non-zero: the records broke the contract and d_a is not sorted).
int fgb_radix_sort_device(void *d_a, void *d_b, long long n, int bit_lo, int bit_hi, int narrow,
                          void *d_tmp, long long tmp_bytes, int *result_in_b, unsigned long long **d_hiflag,
                          void *stream);
int fgb_kmer_bin_shift(long long n, unsigned plo, unsigned phi);
void fgb_kmer_first_digit(long long nmax, unsigned plo, unsigned phi, int *fsh, int *dbits);
long long fgb_kmer_plan_bytes(long long n, unsigned plo, unsigned phi, int fsh, int dbits);
int fgb_kmer_sort_device(void *d_a, void *d_b, long long n, unsigned plo, unsigned phi, int fsh, int dbits,
                         const unsigned long long *d_hist, void *d_tmp, long long tmp_bytes, void *d_plan,
                         int *result_in_b, void *stream);
int fgb_kmer_sort_oversized(const void *src, void *dst, long long n, const void *d_plan, unsigned nover,
                            unsigned ototal, void *stream);

// ---- gix.cu: genome staging, syncmer scan, table index and .ktab entries ----
int fgb_stage_genome_device(const void *d_bps, const long long *d_boff, const long long *d_clen,
                            const long long *d_woff, int ncontig, long long total_words,
                            void *d_seq, void *d_rseq, void *stream);
int fgb_syncmer_digit_count_device(const void *d_seq, const long long *d_clen, const long long *d_woff,
                                   const int *d_crank, const int *d_tile_contig, const int *d_tile_start,
                                   int ntiles, unsigned long long *d_buck1024, unsigned *d_dmat, int dsh, int dbits,
                                   unsigned long long *d_nhist, unsigned long long *d_total, void *d_tmp,
                                   long long tmp_bytes, unsigned plo, unsigned phi, void *stream);
int fgb_syncmer_digit_emit_device(const void *d_seq, const long long *d_clen, const long long *d_woff,
                                  const int *d_crank, const int *d_tile_contig, const int *d_tile_start,
                                  int ntiles, unsigned *d_dmat, int dsh, int dbits, long long n, void *d_records,
                                  unsigned plo, unsigned phi, void *stream);
int fgb_kix_index_device(const void *d_tab, long long n, unsigned *d_pstart, unsigned char *d_adj, void *stream);
int fgb_ktab_export_device(const void *d_tab, long long n, int pbytes, int cbytes,
                           const long long *d_part_first, int nparts, void *d_out, void *stream);
int fgb_ktab_import_device(const void *d_ent, long long n, int pbytes, int cbytes,
                           const long long *d_index, void *d_tab, void *stream);
int fgb_sc_tile();

// ---- merge.cu: adaptamer merge, forward-strand view, seed owners ----
int fgb_forward_view_device(const void *d_T, long long n, void *d_out, long long *h_nfwd, void *stream);
int fgb_self_merge_device(const void *d_T, long long n, const unsigned *d_pstart, int freq,
                          int anti_bits, int band_bits, int jc_bits, int ic_bits,
                          long long amxpos, void *d_seeds, long long capacity,
                          unsigned long long *d_counters, unsigned long long *h_nseeds,
                          unsigned long long *h_sumlen, void *stream);
int fgb_merge_device(const void *d_T1, long long n1, const void *d_T2, long long n2, const unsigned *d_pstart2,
                     const unsigned char *d_adj2, int freq, int anti_bits, int band_bits, int jc_bits, int ic_bits,
                     long long amxpos, long long bmxpos, void *d_seeds, long long capacity,
                     unsigned long long *d_counters, unsigned long long *h_nseeds,
                     unsigned long long *h_sumlen, void *stream);
int fgb_owner_count_device(const void *d_seeds, long long n, int p_ic, int ic_bits, const int *d_owner, int nrc,
                           int world, unsigned long long *d_cnt, void *stream);
int fgb_owner_scatter_device(const void *d_seeds, long long n, int p_ic, int ic_bits, const int *d_owner, int nrc,
                             int world, unsigned long long *d_base, void *d_out, void *stream);

}
