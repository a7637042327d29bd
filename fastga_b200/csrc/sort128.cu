// LSD radix sort of 128-bit records on a bit range of the key, hand-written for sm_90a (H100).
//
// Replaces the reference's two CPU sorts on the hot path:
//   msd_sort   (MSDsort.c:404)  -- k-mer records of the GIX build, key = 40-mer (80 bits)
//   rmsd_sort  (RSDsort.c:292)  -- adaptive-seed records, key = (jcont, band, anti, drem, lcp)
// Both are in-place American-flag MSD sorts on byte-packed records (MSDsort.c:211-360); on the
// device every record is widened to one 16-byte word so each pass is a perfectly coalesced
// stream (read 16 B, write 16 B per record).  One pass = one Onesweep kernel: a stable scatter
// that ranks records inside a tile with a warp multi-split (ballots), finds the tile's bases by
// decoupled look-back, stages the tile in shared memory in digit order and writes digit runs back
// coalesced, while counting the next pass's histogram.  HBM-bound integer work: no tensor cores.
//
// Pass plans (fgb_radix_sort_device):
//   128-bit  every pass reads and writes 16-byte records; the result lands in d_a or d_b.
//   narrow   for records whose hi word is zero (keys of <= 64 bits, two passes or more): the first pass
//            reads the 16-byte records and writes only their lo words (ORing every dropped hi word into
//            a flag), the middle passes run on 8-byte words and the last pass writes 16-byte records
//            again (hi = 0) into d_a: per record 16 + 24 + 16·(passes−2) + 24 bytes instead of
//            16 + 32·passes.
#include "stages.h"
#include <stdlib.h>
#include <utility>
#include <vector>
#include <algorithm>
#include <stdint.h>

#define SORT_THREADS 512
#ifndef SORT_ITEMS
#define SORT_ITEMS   8
#endif
//  items per thread of a pass on 8-byte input: the staging buffer holds one tile of INPUT records,
//  64 KB for both widths, so two CTAs still share an SM
#ifndef SORT64_ITEMS
#define SORT64_ITEMS 16
#endif
#ifndef SORT_MINBLK
#define SORT_MINBLK  2
#endif
#define SORT_TILE    (SORT_THREADS*SORT_ITEMS)
#define SORT_WARPS   (SORT_THREADS/32)
static_assert(SORT_THREADS*SORT64_ITEMS >= SORT_TILE, "fgb_sort128_tmp_bytes sizes the look-back status for SORT_TILE");

typedef unsigned long long u64;

static __device__ __forceinline__ unsigned warp_incl_scan(unsigned v, int lane)
{
#pragma unroll
  for (int o = 1; o < 32; o <<= 1)
    { unsigned t = __shfl_up_sync(0xffffffffu,v,o);
      if (lane >= o) v += t;
    }
  return v;
}

//  the 8-bit digit at bit offset sh of an 8-byte word, and the word's loads and stores, beside the
//  rec128 forms of common.cuh
static __device__ __forceinline__ unsigned rec_dig(u64 v, int sh) { return (unsigned) (v >> sh) & 0xff; }
static __device__ __forceinline__ u64 ld_rec(const u64 *p) { return *p; }
static __device__ __forceinline__ void st_rec(u64 *p, u64 v) { *p = v; }


/***********************************************************************************************
 *  Onesweep pass: one kernel per digit reads every record once and writes it once.
 *   - the GLOBAL digit histogram of a pass is produced by the previous pass (each tile counts
 *     the next digit while it holds the records; the first pass has a small histogram kernel);
 *   - the tile's base inside each digit bucket comes from a decoupled look-back over the
 *     per-tile digit counts (status word = count | flag<<62; 1 = tile aggregate, 2 = inclusive
 *     prefix), tiles being handed out by an atomic ticket so every predecessor is running.
 **********************************************************************************************/

//  Lanes of the warp holding the same 8-bit digit as this lane (among valid lanes).  MATCH.ANY
//  costs one internal round per distinct value in the warp (~30 for random digits); nine ballots
//  are a fixed, much smaller cost.
static __device__ __forceinline__ unsigned match_digit(unsigned d, bool valid)
{ unsigned peers = __ballot_sync(0xffffffffu,valid);
#pragma unroll
  for (int k = 0; k < 8; k++)
    { bool bit = (d >> k) & 1;
      unsigned bk = __ballot_sync(0xffffffffu,bit);
      peers &= bit ? bk : ~bk;
    }
  return peers;
}

//  Rank of this lane's item among the items of digit d its warp has ranked so far: myc is the warp's
//  count column (myc[d] = items of digit d in earlier rounds), bumped by the round's leader.
static __device__ __forceinline__ unsigned warp_rank(unsigned *myc, unsigned d, bool valid)
{ const int lane = threadIdx.x & 31;
  unsigned peers = match_digit(d,valid);
  int leader = valid ? __ffs(peers)-1 : lane;
  unsigned b = 0;
  if (valid && lane == leader)
    { b = myc[d];
      myc[d] = b + __popc(peers);
    }
  b = __shfl_sync(0xffffffffu,b,leader);
  __syncwarp();
  return b + __popc(peers & lanemask_lt());
}

//  Once every warp has ranked its items: wcount[w][d] (the count columns, SORT_WARPS x 256) becomes the
//  count of digit d in the warps before w, and bexcl[d] the tile's count of the digits below d.  Thread
//  d < 256 returns the tile's count of digit d and hands it to publish before the scan.  Ends on a barrier.
template <class F>
static __device__ __forceinline__ unsigned digit_offsets(unsigned *wcount, unsigned *bexcl, unsigned *wtot, F publish)
{ const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  unsigned c = 0, inc = 0;
  __syncthreads();
  if (tid < 256)
    {
#pragma unroll
      for (int ww = 0; ww < SORT_WARPS; ww++)
        { unsigned t = wcount[ww*256+tid];
          wcount[ww*256+tid] = c;
          c += t;
        }
      publish(c);
      inc = warp_incl_scan(c,lane);
      if (lane == 31) wtot[w] = inc;
    }
  __syncthreads();
  if (tid < 256)
    { unsigned pre = 0;
      for (int i = 0; i < w; i++) pre += wtot[i];
      bexcl[tid] = pre + inc - c;
    }
  __syncthreads();
  return c;
}

#define ST_AGG  (1ull << 62)
#define ST_INC  (2ull << 62)
#define ST_MASK ((1ull << 62) - 1)

//  Records of digit d (d = tid < 256) in the tiles before tileid.  Four predecessors per round trip:
//  the status words of consecutive tiles are independent loads, a serial walk pays one L2 latency per
//  tile, and the walk is as deep as the tiles in flight.  A tile that has published nothing yet is
//  read again from there on.
static __device__ __forceinline__ u64 lookback(const u64 *status, unsigned tileid, int tid)
{ volatile const u64 *stt = status;
  u64 excl = 0;
  for (long long t = (long long) tileid - 1; t >= 0; )
    { u64 v[4];
#pragma unroll
      for (int q = 0; q < 4; q++)
        v[q] = (t - q >= 0) ? stt[(u64) (t - q)*256 + tid] : ST_INC;
      bool done = false;
#pragma unroll
      for (int q = 0; q < 4; q++)
        { if (done || (v[q] >> 62) == 0) break;
          excl += v[q] & ST_MASK;
          t -= 1;
          if (v[q] & ST_INC) done = true;
        }
      if (done) break;
    }
  return excl;
}

__global__ void __launch_bounds__(SORT_THREADS)
sort_ghist_kernel(const rec128 *__restrict__ in, long long n, int dsh /* digit = bits [dsh,dsh+8) */, unsigned long long *__restrict__ ghist)
{ __shared__ unsigned h[256];
  int tid = threadIdx.x;
  if (tid < 256) h[tid] = 0;
  __syncthreads();
  //  a digit inside one 64-bit half is counted from that half alone (half the traffic)
  const bool one = (dsh >= 64 || dsh <= 56);
  const unsigned long long *half = reinterpret_cast<const unsigned long long *>(in) + (dsh >= 64);
  const int sh = dsh & 63;
  for (long long tile0 = (long long) blockIdx.x * SORT_TILE; tile0 < n; tile0 += (long long) gridDim.x * SORT_TILE)
    {
#pragma unroll
      for (int it = 0; it < SORT_ITEMS; it++)
        { long long idx = tile0 + it*SORT_THREADS + tid;
          bool valid = idx < n;
          unsigned d = 0;
          if (valid) d = one ? (unsigned) ((half[2*idx] >> sh) & 0xff) : rec_dig(ld_rec(in + idx),dsh);
          unsigned peers = match_digit(d,valid);             // one atomic per distinct digit of the warp
          if (valid && (tid & 31) == __ffs(peers)-1) atomicAdd(&h[d],__popc(peers));
        }
    }
  __syncthreads();
  if (tid < 256 && h[tid]) atomicAdd(&ghist[tid],(unsigned long long) h[tid]);
}

//  exclusive scan of a 256-bin global histogram -> bin bases; zeroes the histogram of the pass
//  after it and the tile ticket.
__global__ void sort_bins_kernel(const unsigned long long *__restrict__ ghist, unsigned long long *__restrict__ binbase,
                                 unsigned long long *__restrict__ nexthist, unsigned *__restrict__ ticket)
{ __shared__ unsigned long long ws[8];
  int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  unsigned long long v = ghist[tid], inc = v;
  for (int o = 1; o < 32; o <<= 1)
    { unsigned long long t = __shfl_up_sync(0xffffffffu,inc,o);
      if (lane >= o) inc += t;
    }
  if (lane == 31) ws[w] = inc;
  __syncthreads();
  unsigned long long pre = 0;
  for (int i = 0; i < w; i++) pre += ws[i];
  binbase[tid] = pre + inc - v;
  nexthist[tid] = 0;
  if (tid == 0) *ticket = 0;
}

//  IW: bytes per input record; a tile holds SORT_ITEMS 16-byte records or SORT64_ITEMS 8-byte words per thread
template <int IW> struct os_tile
{ static constexpr int ITEMS = (IW == 16) ? SORT_ITEMS : SORT64_ITEMS;
  static constexpr int TILE  = SORT_THREADS*ITEMS;
  static constexpr size_t SMEM = (size_t) TILE*IW + (SORT_WARPS*256 + 256 + 256 + 8)*sizeof(unsigned)
                                 + 256*sizeof(u64);
};

//  One pass on the digit at bit dsh.  Key: the word ranked and held in registers, a rec128 or the lo
//  word of a record whose hi word must be zero.  IW / OW: bytes per input / output record.  A 16-byte
//  record read into a u64 Key ORs its hi word into *hiflag; a u64 Key written as 16 bytes gets hi = 0.
template <class Key, int IW, int OW>
__global__ void __launch_bounds__(SORT_THREADS,SORT_MINBLK)
sort_onesweep_kernel(const void *__restrict__ in, void *__restrict__ out, long long n, int dsh /* bit offset of the digit */,
                     int next_dsh /* of the next pass's digit, -1: none */, const u64 *__restrict__ binbase,
                     u64 *__restrict__ nexthist, u64 *status /* [ntiles][256] */, unsigned *__restrict__ ticket,
                     u64 *__restrict__ hiflag)
{ constexpr int ITEMS = os_tile<IW>::ITEMS, TILE = os_tile<IW>::TILE;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Key      *tile   = reinterpret_cast<Key *>(smem_raw);                  // input tile, then the keys in digit order
  unsigned *wcount = reinterpret_cast<unsigned *>(smem_raw + (size_t) TILE*IW); // [SORT_WARPS][256]
  unsigned *bexcl  = wcount + SORT_WARPS*256;                           // [256]
  unsigned *nhist  = bexcl + 256;                                       // [256] next digit
  unsigned *wtot   = nhist + 256;                                       // [8]
  u64      *gbase  = reinterpret_cast<u64 *>(wtot + 8);                 // [256]
  __shared__ unsigned tile_s;
  __shared__ __align__(8) u64 tbar;

  int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (tid == 0)
    { unsigned t = atomicAdd(ticket,1u);
      tile_s = t;
      //  the tile's consecutive input records: fetched by one TMA bulk copy (UBLKCP) into the staging
      //  buffer while the block zeroes its counters.  An odd count of 8-byte words is rounded up to the
      //  16 bytes a bulk copy moves (the caller's buffers have room for that word; it is never ranked).
      long long t0 = (long long) t * TILE, rm = n - t0;
      unsigned nb = ((unsigned) (rm < TILE ? rm : TILE) * IW + 15u) & ~15u;
      mbar_init(&tbar,1);
      tma_load_1d(tile,reinterpret_cast<const unsigned char *>(in) + t0*IW,nb,&tbar);
    }
  for (int i = tid; i < SORT_WARPS*256; i += SORT_THREADS) wcount[i] = 0;
  if (tid < 256) nhist[tid] = 0;
  __syncthreads();
  const unsigned tileid = tile_s;
  long long tile0 = (long long) tileid * TILE;
  long long rem = n - tile0;
  int cnt = rem < TILE ? (int) rem : TILE;

  Key      r[ITEMS];
  unsigned rank[ITEMS];
  u64      hi_or = 0;
  int base = w*(32*ITEMS);
  unsigned *myc = wcount + w*256;
  mbar_wait(&tbar,0);
#pragma unroll
  for (int it = 0; it < ITEMS; it++)
    { int idx = base + it*32 + lane;
      bool valid = idx < cnt;
      unsigned d = 0;
      if (valid)
        { if constexpr (sizeof(Key) < IW)
            { rec128 v = ld_rec(reinterpret_cast<const rec128 *>(smem_raw) + idx);
              r[it] = v.lo;
              hi_or |= v.hi;
            }
          else
            r[it] = ld_rec(tile + idx);
          d = rec_dig(r[it],dsh);
        }
      rank[it] = warp_rank(myc,d,valid);
      if (next_dsh >= 0 && valid) atomicAdd(&nhist[rec_dig(r[it],next_dsh)],1u);
    }
  if (sizeof(Key) < IW && hi_or) atomicOr(hiflag,hi_or);

  //  Order of the rest: publish the tile's digit counts at once (the tiles after this one add them up
  //  while it works on), place the records in digit order inside the tile, and only THEN look back for
  //  this tile's own bases -- by which time the tiles before it have had the whole placement phase to
  //  publish theirs, so the walk is short and rarely spins.
  u64 *mine = status + (u64) tileid*256 + tid;
  const unsigned c = digit_offsets(wcount,bexcl,wtot,[&](unsigned total)
    { if (tileid == 0)
        atomicExch(mine,ST_INC | total);
      else
        atomicExch(mine,ST_AGG | total);
    });

#pragma unroll
  for (int it = 0; it < ITEMS; it++)
    { int idx = base + it*32 + lane;
      if (idx < cnt)
        { unsigned d = rec_dig(r[it],dsh);
          st_rec(tile + (bexcl[d] + myc[d] + rank[it]),r[it]);
        }
    }
  if (tid < 256)
    { u64 excl = lookback(status,tileid,tid);
      if (tileid != 0) atomicExch(mine,ST_INC | (excl + c));
      gbase[tid] = binbase[tid] + excl - bexcl[tid];
      if (next_dsh >= 0 && nhist[tid]) atomicAdd(&nexthist[tid],(u64) nhist[tid]);
    }
  __syncthreads();

  for (int p = tid; p < cnt; p += SORT_THREADS)
    { Key v = ld_rec(tile + p);
      u64 o = gbase[rec_dig(v,dsh)] + p;
      if constexpr (sizeof(Key) < OW)
        { rec128 R; R.lo = v; R.hi = 0;
          st_rec(reinterpret_cast<rec128 *>(out) + o,R);
        }
      else
        st_rec(reinterpret_cast<Key *>(out) + o,v);
    }
}

//  The tmp block of a sort (fgb_sort128_tmp_bytes): the look-back status words of a pass (256 per tile
//  of SORT_TILE records, the smallest tile), the histograms of this pass's digit and the next one, the
//  bin bases, and a 16-word slot that holds the tile ticket (word 0) and the flag of dropped hi words
//  (word 1).
struct sort_tmp
{ u64 *status, *hist[2], *binbase, *hiflag;
  unsigned *ticket;
  sort_tmp(void *d_tmp, long long n)
    { long long ntiles = (n + SORT_TILE - 1) / SORT_TILE;
      if (ntiles < 1) ntiles = 1;
      status  = (u64 *) d_tmp;
      hist[0] = status + 256ull*ntiles;
      hist[1] = hist[0] + 256;
      binbase = hist[1] + 256;
      ticket  = (unsigned *) (binbase + 256);
      hiflag  = binbase + 256 + 1;
    }
};

extern "C" long long fgb_sort128_tmp_bytes(long long n)
{ long long ntiles = (n + SORT_TILE - 1) / SORT_TILE;
  if (ntiles < 1) ntiles = 1;
  return 256*ntiles*8 + (3*256 + 16)*8;
}

//  The histogram of the first pass's digit, bits [dsh, dsh+8) of the n records in d_a, into T.hist[0].
static int first_pass_hist(const void *d_a, long long n, int dsh, const sort_tmp &T, cudaStream_t st)
{ CUDA_TRY(cudaMemsetAsync(T.hist[0],0,256*8,st));
  int ntiles = (int) ((n + SORT_TILE - 1) / SORT_TILE), nb = ntiles < 1184 ? ntiles : 1184;
  sort_ghist_kernel<<<nb,SORT_THREADS,0,st>>>((const rec128 *) d_a,n,dsh,T.hist[0]);
  fgb_count_launch(1);
  return FGB_OK;
}

//  One pass: the bin bases of this pass's histogram (cur), the status words zeroed, the Onesweep kernel.
template <class Key, int IW, int OW>
static int onesweep_pass(const void *in, void *out, long long n, int dsh, int next_dsh, const sort_tmp &T, int cur,
                         cudaStream_t st)
{ typedef os_tile<IW> O;
  static bool attr_set = false;
  if (!attr_set)
    { CUDA_TRY(cudaFuncSetAttribute(sort_onesweep_kernel<Key,IW,OW>,cudaFuncAttributeMaxDynamicSharedMemorySize,(int) O::SMEM));
      attr_set = true;
    }
  int ntiles = (int) ((n + O::TILE - 1) / O::TILE);
  sort_bins_kernel<<<1,256,0,st>>>(T.hist[cur],T.binbase,T.hist[cur^1],T.ticket);
  CUDA_TRY(cudaMemsetAsync(T.status,0,256ull*ntiles*8,st));
  sort_onesweep_kernel<Key,IW,OW><<<ntiles,SORT_THREADS,O::SMEM,st>>>(in,out,n,dsh,next_dsh,T.binbase,T.hist[cur^1],
                                                                     T.status,T.ticket,T.hiflag);
  fgb_count_launch(2);
  return FGB_OK;
}

extern "C" int fgb_radix_sort_device(void *d_a, void *d_b, long long n, int bit_lo, int bit_hi, int narrow,
                                     void *d_tmp, long long tmp_bytes, int *result_in_b, u64 **d_hiflag, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (n < 0 || bit_lo < 0 || bit_hi > (narrow ? 64 : 128) || bit_lo > bit_hi) return FGB_ERR_ARG;
  if (n >= 0xffffffffll) return FGB_ERR_LIMIT;
  *result_in_b = 0;
  const sort_tmp T(d_tmp,n);
  if (narrow)                                 // the caller reads the flag whether or not anything is sorted
    { if (tmp_bytes < fgb_sort128_tmp_bytes(n)) return FGB_ERR_ARG;
      CUDA_TRY(cudaMemsetAsync(T.hiflag,0,8,st));
      *d_hiflag = T.hiflag;
    }
  if (n <= 1 || bit_lo == bit_hi) return FGB_OK;
  if (tmp_bytes < fgb_sort128_tmp_bytes(n)) return FGB_ERR_ARG;

  const int npass = (bit_hi - bit_lo + 7) / 8;
  const bool words = narrow && npass >= 2;    // one pass: nothing to narrow, the 128-bit pass runs
  //  the two 8-byte ping-pong buffers of the narrow plan are the two halves of d_b (16(n+1) bytes); the
  //  second half starts 16-byte aligned, and both may be read one word past their end
  void *half[2] = { d_b, (unsigned char *) d_b + ((8*n + 15) & ~15ll) };

  int rc = first_pass_hist(d_a,n,bit_lo,T,st);
  for (int p = 0; p < npass && rc == FGB_OK; p++)
    { const int b = bit_lo + 8*p, nd = (p + 1 < npass) ? b + 8 : -1, cur = p & 1;
      if (!words)
        rc = onesweep_pass<rec128,16,16>(cur ? d_b : d_a,cur ? d_a : d_b,n,b,nd,T,cur,st);
      else if (p == 0)
        rc = onesweep_pass<u64,16,8>(d_a,half[0],n,b,nd,T,cur,st);
      else if (nd >= 0)
        rc = onesweep_pass<u64,8,8>(half[cur^1],half[cur],n,b,nd,T,cur,st);
      else
        rc = onesweep_pass<u64,8,16>(half[cur^1],d_a,n,b,nd,T,cur,st);
    }
  if (rc) return rc;
  CUDA_TRY(cudaGetLastError());
  if (!words && (npass & 1))
    { if (narrow)
        CUDA_TRY(cudaMemcpyAsync(d_a,d_b,sizeof(rec128)*n,cudaMemcpyDeviceToDevice,st));
      else
        *result_in_b = 1;
    }
  return FGB_OK;
}

extern "C" int fgb_sort128_device(void *d_a, void *d_b, long long n, int byte_lo, int byte_hi,
                                  void *d_tmp, long long tmp_bytes, int *result_in_b, void *stream)
{ if (byte_lo < 0 || byte_hi > 16 || byte_lo > byte_hi) return FGB_ERR_ARG;
  return fgb_radix_sort_device(d_a,d_b,n,8*byte_lo,8*byte_hi,0,d_tmp,tmp_bytes,result_in_b,NULL,stream);
}

/***********************************************************************************************
 *  k-mer table sort (msd_sort's job in GIXmake.c:1436): by the 40-mer (bytes 6..15), equal
 *  k-mers by (strand|contig rank, post), i.e. by the whole 128-bit value.
 *
 *  Ten full Onesweep passes move 10 x 32 bytes per record through HBM.  Instead:
 *    1. the records are laid out by prefix bin: bin p at [bins[p], bins[p+1]), in any order inside
 *       the bin.  Onesweep partition passes on the prefix bits above the bin shift give that
 *       layout (fgb_kmer_sort_device).  A table built from a genome gets its lowest digit from the
 *       scan itself: the scan's emit pass stores the records in runs by that digit;
 *    2. the bins' starts are found on the device and consecutive bins packed there into groups of at
 *       most BK_CAP records and BK_SPAN bins (kmer_fine_bounds_kernel, kmer_plan_kernel); a CTA pulls a
 *       group into shared memory with one TMA bulk copy, sorts it there (kmer_bucket_sort_kernel) and
 *       writes it back once;
 *    3. bins larger than BK_CAP (repeats) are compacted, sorted with the generic Onesweep sort and
 *       copied back (fgb_kmer_sort_oversized, once the host has read the plan's count of them).
 *  Every record is unique (contig, strand and post differ) and steps 2 and 3 order a bin by the whole
 *  128-bit value, so the order records arrive in inside a bin does not change the table.
 *  HBM traffic per record after the layout: 32 bytes (10 x 32 for a full LSD sort).
 **********************************************************************************************/

#define BK_THREADS SORT_THREADS
#define BK_ITEMS   8
#define BK_CAP     (BK_THREADS*BK_ITEMS)
#define BK_WARPS   SORT_WARPS
#define BK_SPAN    4                     // a group covers at most this many consecutive 16-bit bins
#define BK_SUBBITS 10
#define BK_NSUB    (BK_SPAN << BK_SUBBITS)
#define BK_MAXSUB  32                    // a sub-bin longer than this sends the group down the LSD path

//  fstart[p] = first record whose fine bin ((hi >> binshift) - base) is >= p, p in [0,nf]: a lower-bound search
//  over the partitioned records, whose fine bins never decrease.  About log2(n) 8-byte probes per fine bin, most of
//  them shared with the neighbouring threads' searches, instead of a pass over all 16 n bytes.
__global__ void kmer_fine_bounds_kernel(const rec128 *__restrict__ tab, long long n, int binshift, unsigned long long base,
                                        unsigned *__restrict__ fstart, long long nf)
{ long long p = (long long) blockIdx.x * blockDim.x + threadIdx.x;
  if (p > nf) return;
  long long lo = 0, hi = n;
  while (lo < hi)
    { long long md = (lo + hi) >> 1;
      if ((tab[md].hi >> binshift) - base < (unsigned long long) p) lo = md + 1; else hi = md;
    }
  fstart[p] = (unsigned) lo;
}

//  The plan of a k-mer sort (fgb_kmer_plan_bytes): counters, the oversized bins, the fine-bin starts and the groups.
#define KP_NGROUPS 0                      // counter words: groups, oversized bins, records in oversized bins
#define KP_NOVER   1
#define KP_OTOTAL  2
struct kmer_plan
{ unsigned *ctr, *fstart;
  uint2 *over;                            // oversized bins: start, length (in no particular order)
  uint4 *groups;                          // start, count, hi >> binshift of the first bin (in no particular order)
  kmer_plan(void *d, long long n, long long nf)
    { long long ocap = n / BK_CAP + 1;
      ctr = (unsigned *) d;
      over = (uint2 *) (ctr + 4);
      fstart = (unsigned *) (over + ocap);
      groups = (uint4 *) (((uintptr_t) (fstart + nf + 1) + 15) & ~(uintptr_t) 15);
    }
};

//  One thread per window of BK_SPAN consecutive bins packs the window's bins greedily into groups: whole bins, at
//  most BK_CAP records (a window never exceeds BK_SPAN bins).  Bins larger than BK_CAP go to the oversized list.
//  Bin p starts at the first of its fine bins, fstart[((base + p) << dsh) - fbase].
__global__ void kmer_plan_kernel(long long nf, long long nbins, int dsh, unsigned long long base,
                                 unsigned long long fbase, kmer_plan P)
{ long long p0 = ((long long) blockIdx.x * blockDim.x + threadIdx.x) * BK_SPAN;
  if (p0 >= nbins) return;
  const int nb = nbins - p0 < BK_SPAN ? (int) (nbins - p0) : BK_SPAN;
  unsigned b[BK_SPAN+1];
#pragma unroll
  for (int k = 0; k <= BK_SPAN; k++)
    if (k <= nb)
      { long long f = (long long) ((base + p0 + k) << dsh) - (long long) fbase;
        b[k] = P.fstart[f < 0 ? 0 : (f > nf ? nf : f)];
      }
  uint4 g[BK_SPAN];
  int ng = 0;
  unsigned gs = 0, gc = 0, gp = 0;
#pragma unroll
  for (int k = 0; k < BK_SPAN; k++)
    { if (k >= nb) break;
      unsigned len = b[k+1] - b[k];
      if (len == 0) continue;
      if (len > BK_CAP)
        { if (gc) { g[ng++] = make_uint4(gs,gc,(unsigned) (base + p0) + gp,0); gc = 0; }
          P.over[atomicAdd(&P.ctr[KP_NOVER],1u)] = make_uint2(b[k],len);
          atomicAdd(&P.ctr[KP_OTOTAL],len);
          continue;
        }
      if (gc + len > BK_CAP) { g[ng++] = make_uint4(gs,gc,(unsigned) (base + p0) + gp,0); gc = 0; }
      if (gc == 0) { gs = b[k]; gp = k; }
      gc += len;
    }
  if (gc) g[ng++] = make_uint4(gs,gc,(unsigned) (base + p0) + gp,0);
  if (ng == 0) return;
  unsigned o = atomicAdd(&P.ctr[KP_NGROUPS],(unsigned) ng);
  for (int k = 0; k < ng; k++) P.groups[o+k] = g[k];
}

//  Each CTA sorts groups blockIdx.x, blockIdx.x + gridDim.x, ... of the *ngroups groups (<= BK_CAP records of <=
//  BK_SPAN consecutive bins each) by the full 128-bit value.  Fast path: a counting split on the next 10 key bits
//  (shared-memory atomics) leaves sub-bins of one or two records, and every record finds its place by comparing
//  itself with its sub-bin.  A group with a crowded sub-bin (repeats) runs sixteen LSD byte passes instead.

__global__ void __launch_bounds__(BK_THREADS,2)
kmer_bucket_sort_kernel(const rec128 *__restrict__ in, rec128 *__restrict__ out,
                        const uint4 *__restrict__ groups /* start, count, hi >> binshift of its first bin */,
                        const unsigned *__restrict__ ngroups, int binshift)
{ extern __shared__ __align__(16) unsigned char smem_raw[];
  rec128   *tile   = reinterpret_cast<rec128 *>(smem_raw);
  unsigned *cnt    = reinterpret_cast<unsigned *>(tile + BK_CAP);        // [BK_NSUB+1]; LSD path: wcount[BK_WARPS][256]
  unsigned *bexcl  = cnt + BK_NSUB + 32;                                  // [256]
  unsigned *wtot   = bexcl + 256;                                         // [BK_WARPS]
  __shared__ __align__(8) unsigned long long tbar;

  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const unsigned ng = *ngroups;
  if (blockIdx.x >= ng) return;
  if (tid == 0) mbar_init(&tbar,1);
  unsigned phase = 0;
  for (unsigned gi = blockIdx.x; gi < ng; gi += gridDim.x, phase ^= 1)
    {
    const uint4 g = groups[gi];
    const int count = (int) g.y;
    if (tid == 0)
      { asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the last group's stores before the copy
        tma_load_1d(tile,in + g.x,(unsigned) count * 16u,&tbar);
      }
    for (int i = tid; i <= BK_NSUB; i += BK_THREADS) cnt[i] = 0;
    __syncthreads();
    mbar_wait(&tbar,phase);

    rec128   r[BK_ITEMS];
    unsigned sub[BK_ITEMS], off[BK_ITEMS];
    const int base = w*(32*BK_ITEMS);
    const unsigned b0 = g.z;                     // not tile[0]'s bin: a bin's records come in any order
    const int subshift = binshift - BK_SUBBITS;
#pragma unroll
    for (int it = 0; it < BK_ITEMS; it++)
      { int idx = base + it*32 + lane;
        if (idx < count)
          { r[it] = ld_rec(tile + idx);
            sub[it] = ((((unsigned) (r[it].hi >> binshift)) - b0) << BK_SUBBITS) | ((unsigned) (r[it].hi >> subshift) & ((1u << BK_SUBBITS)-1));
            off[it] = atomicAdd(&cnt[sub[it]],1u);
          }
      }
    __syncthreads();
    //  exclusive scan of the sub-bin counts (8 per thread), crowded sub-bin detection
    bool big = false;
    { unsigned v[8], sum = 0;
#pragma unroll
      for (int i = 0; i < 8; i++) { v[i] = cnt[8*tid+i]; big |= (v[i] > BK_MAXSUB); sum += v[i]; }
      unsigned inc = warp_incl_scan(sum,lane);
      if (lane == 31) wtot[w] = inc;
      __syncthreads();
      unsigned pre = inc - sum;
      for (int i = 0; i < w; i++) pre += wtot[i];
#pragma unroll
      for (int i = 0; i < 8; i++) { cnt[8*tid+i] = pre; pre += v[i]; }
      if (tid == BK_THREADS-1) cnt[BK_NSUB] = pre;
    }
    big = __syncthreads_or(big);

    if (!big)
      {
#pragma unroll
        for (int it = 0; it < BK_ITEMS; it++)
          { int idx = base + it*32 + lane;
            if (idx < count) st_rec(tile + (cnt[sub[it]] + off[it]),r[it]);
          }
        __syncthreads();
        for (int p = tid; p < count; p += BK_THREADS)
          { rec128 R = ld_rec(tile + p);
            unsigned sb = ((((unsigned) (R.hi >> binshift)) - b0) << BK_SUBBITS) | ((unsigned) (R.hi >> subshift) & ((1u << BK_SUBBITS)-1));
            int s = (int) cnt[sb], e = (int) cnt[sb+1], rank = 0;
            for (int q = s; q < e; q++)
              { rec128 Q = ld_rec(tile + q);
                bool less = (Q.hi < R.hi) || (Q.hi == R.hi && (Q.lo < R.lo || (Q.lo == R.lo && q < p)));
                rank += less;
              }
            st_rec(out + (g.x + s + rank),R);
          }
        __syncthreads();
        continue;
      }

    //  LSD path: all sixteen bytes, records still in registers in load order
    unsigned *wcount = cnt;
    unsigned *myc = wcount + w*256;
    unsigned rank[BK_ITEMS];
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 8; i++) myc[i*32 + lane] = 0;
    __syncwarp();
    for (int byte = 0; byte < 16; byte++)
      {
#pragma unroll
        for (int it = 0; it < BK_ITEMS; it++)
          { int idx = base + it*32 + lane;
            bool valid = idx < count;
            rank[it] = warp_rank(myc,valid ? rec_byte(r[it],byte) : 0,valid);
          }
        digit_offsets(wcount,bexcl,wtot,[](unsigned) {});
#pragma unroll
        for (int it = 0; it < BK_ITEMS; it++)
          { int idx = base + it*32 + lane;
            if (idx < count)
              { unsigned d = rec_byte(r[it],byte);
                st_rec(tile + (bexcl[d] + myc[d] + rank[it]),r[it]);
              }
          }
        __syncthreads();
        if (byte + 1 < 16)
          {
#pragma unroll
            for (int it = 0; it < BK_ITEMS; it++)
              { int idx = base + it*32 + lane;
                if (idx < count) r[it] = ld_rec(tile + idx);
              }
#pragma unroll
            for (int i = 0; i < 8; i++) myc[i*32 + lane] = 0;
            __syncwarp();
          }
      }
    for (int p = tid; p < count; p += BK_THREADS)
      st_rec(out + (g.x + p),ld_rec(tile + p));
    __syncthreads();
    }
}

//  copies record segments: src[sfrom[k] .. +len[k]) -> dst[dfrom[k] ..); pre[] = prefix sums of len
__global__ void kmer_copy_segments_kernel(const rec128 *__restrict__ src, rec128 *__restrict__ dst,
                                          const unsigned *__restrict__ sfrom, const unsigned *__restrict__ dfrom,
                                          const unsigned *__restrict__ pre, int nseg, long long total)
{ for (long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long) gridDim.x * blockDim.x)
    { int lo = 0, hi = nseg;                                  // last k with pre[k] <= i
      while (hi - lo > 1) { int md = (lo+hi) >> 1; if (pre[md] <= i) lo = md; else hi = md; }
      unsigned o = (unsigned) (i - pre[lo]);
      st_rec(dst + (dfrom[lo] + o),ld_rec(src + (sfrom[lo] + o)));
    }
}

static const size_t BUCKET_SMEM = BK_CAP*sizeof(rec128) + (BK_NSUB + 32 + 256 + BK_WARPS)*sizeof(unsigned);

//  The bins of n records whose 12-base prefixes lie in [plo,phi) (the whole space, or one rank's share
//  of a cooperatively built table): bin = (prefix24 >> sh) - (plo >> sh).  The bins always tile THAT
//  range, so a share is binned as finely as a whole table of the same size.  As many bins as keep the
//  average bin near 1.5 K records (a CTA sorts <= BK_CAP in shared memory): 65536 up to ~100 M records,
//  one more power of two per doubling beyond (a 1 Gbp genome: 2^19).  sh never grows with n, so the
//  bins chosen for an upper bound of n refine the bins chosen for n.
extern "C" int fgb_kmer_bin_shift(long long n, unsigned plo, unsigned phi)
{ long long maxbins = 65536, target = 1536;
  if (getenv("FGB_KSORT_BIN_TARGET") != NULL) target = atoll(getenv("FGB_KSORT_BIN_TARGET"));   // tests: force more bins
  if (target < 1) target = 1;
  while (maxbins < (1ll << 24) && n / maxbins > target) maxbins <<= 1;
  int sh = 0;
  while ((long long) ((((unsigned long long) (phi - 1) >> sh) - ((unsigned long long) plo >> sh))) >= maxbins) sh += 1;
  return sh;
}

//  The k-mer partition a table's syncmer scan starts: the partition sorts bits [fsh, 24) of the 12-base
//  prefix, fsh chosen for an upper bound nmax of n, by a first digit of dbits bits that the scan's emit pass
//  lays out and 8-bit Onesweep passes above it.  The first digit takes what is left over by as few passes
//  as leave it at most 9 bits.
extern "C" void fgb_kmer_first_digit(long long nmax, unsigned plo, unsigned phi, int *fsh, int *dbits)
{ *fsh = fgb_kmer_bin_shift(nmax,plo,phi);
  int bits = 24 - *fsh, passes = (bits - 9 + 7) / 8;
  if (passes < 1) passes = 1;
  *dbits = bits - 8*passes;
}

//  The bins of the rule for n (fgb_kmer_bin_shift) and the fine bins the partition passes lay out
static void kmer_bins_of(long long n, unsigned plo, unsigned phi, int *fsh, int dbits, int *sh, long long *nf,
                         long long *nbins)
{ *sh = fgb_kmer_bin_shift(n,plo,phi);
  if (dbits == 0) *fsh = *sh;
  *nf = (long long) (((unsigned long long) (phi - 1) >> *fsh) - ((unsigned long long) plo >> *fsh)) + 1;
  *nbins = (long long) (((unsigned long long) (phi - 1) >> *sh) - ((unsigned long long) plo >> *sh)) + 1;
}

//  Bytes of the plan block of fgb_kmer_sort_device
extern "C" long long fgb_kmer_plan_bytes(long long n, unsigned plo, unsigned phi, int fsh, int dbits)
{ int sh;
  long long nf = 1, nbins = 1;
  if (phi > plo) kmer_bins_of(n,plo,phi,&fsh,dbits,&sh,&nf,&nbins);
  return 16 + 8*(n / BK_CAP + 1) + 4*(nf + 1) + 16 + 16*nbins;
}

//  Sorts the n records in d_a whose 12-base prefixes lie in [plo,phi); d_b: scratch of the same size, d_tmp as
//  for fgb_sort128_device, d_plan a block of fgb_kmer_plan_bytes.  The sorted table lands in d_a or d_b
//  (*result_in_b).  Onesweep passes on the prefix above bit fsh lay the records out by fine bin,
//  (prefix24 >> fsh) - (plo >> fsh); a bin of the rule for n is a run of whole fine bins, so the records then go
//  straight to the bucket sort.
//    dbits > 0: the syncmer scan laid d_a out by the first digit of the partition, bits [fsh, fsh+dbits) of
//      the prefix (fgb_kmer_first_digit, fsh chosen for an upper bound of n), and d_hist holds the histogram
//      of the 8 prefix bits above it.
//    dbits = 0: the records are in any order; fsh is the bin shift for n, and the first pass counts its own
//      histogram.
//  Does not synchronise: the fine-bin starts and the bucket-sort groups are planned on the device.  The bins
//  larger than BK_CAP are left out of the result: the plan's first four words (KP_*) count them, and when
//  there are any, fgb_kmer_sort_oversized puts them in place.
extern "C" int fgb_kmer_sort_device(void *d_a, void *d_b, long long n, unsigned plo, unsigned phi, int fsh, int dbits,
                                    const u64 *d_hist, void *d_tmp, long long tmp_bytes, void *d_plan,
                                    int *result_in_b, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  *result_in_b = 0;
  CUDA_TRY(cudaMemsetAsync(d_plan,0,16,st));
  if (n <= 1) return FGB_OK;
  if (n >= 0xffffffffll) return FGB_ERR_LIMIT;
  if (phi <= plo || phi > (1u << 24) || tmp_bytes < fgb_sort128_tmp_bytes(n)) return FGB_ERR_ARG;
  int sh;
  long long nf, nbins;
  kmer_bins_of(n,plo,phi,&fsh,dbits,&sh,&nf,&nbins);
  if (sh < fsh) return FGB_ERR_ARG;
  const sort_tmp T(d_tmp,n);
  const int b0 = 64 + 40 + fsh + dbits, npass = (128 - b0 + 7) / 8;
  if (dbits == 0)
    { int rc = first_pass_hist(d_a,n,b0,T,st);
      if (rc) return rc;
    }
  else
    CUDA_TRY(cudaMemcpyAsync(T.hist[0],d_hist,256*8,cudaMemcpyDeviceToDevice,st));
  rec128 *src = (rec128 *) d_a, *dst = (rec128 *) d_b;
  for (int p = 0; p < npass; p++)
    { const int b = b0 + 8*p, nd = (p + 1 < npass) ? b + 8 : -1;
      int rc = onesweep_pass<rec128,16,16>(src,dst,n,b,nd,T,p & 1,st);
      if (rc) return rc;
      std::swap(src,dst);
    }

  static int grid = 0;
  if (grid == 0)
    { int dev, nsm, per;
      CUDA_TRY(cudaFuncSetAttribute(kmer_bucket_sort_kernel,cudaFuncAttributeMaxDynamicSharedMemorySize,(int) BUCKET_SMEM));
      CUDA_TRY(cudaGetDevice(&dev));
      CUDA_TRY(cudaDeviceGetAttribute(&nsm,cudaDevAttrMultiProcessorCount,dev));
      CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per,kmer_bucket_sort_kernel,BK_THREADS,BUCKET_SMEM));
      grid = nsm * (per > 0 ? per : 1);
    }
  const kmer_plan P(d_plan,n,nf);
  const unsigned long long base = (unsigned long long) plo >> sh, fbase = (unsigned long long) plo >> fsh;
  const long long nwin = (nbins + BK_SPAN - 1) / BK_SPAN;
  kmer_fine_bounds_kernel<<<(int) ((nf + 1 + 255) / 256),256,0,st>>>(src,n,40 + fsh,fbase,P.fstart,nf);
  kmer_plan_kernel<<<(int) ((nwin + 255) / 256),256,0,st>>>(nf,nbins,sh - fsh,base,fbase,P);
  kmer_bucket_sort_kernel<<<(unsigned) (nbins < grid ? nbins : grid),BK_THREADS,BUCKET_SMEM,st>>>(src,dst,P.groups,
                                                                                                  P.ctr + KP_NGROUPS,
                                                                                                  40 + sh);
  fgb_count_launch(3);
  CUDA_TRY(cudaGetLastError());
  *result_in_b = (dst == (rec128 *) d_b);
  return FGB_OK;
}

//  The bins the plan of fgb_kmer_sort_device found larger than BK_CAP (nover bins, ototal records: the plan's
//  KP_NOVER and KP_OTOTAL words): compacted, sorted with the Onesweep sort and copied from the partitioned
//  records (src, the side the result did not land in) into place in the table (dst).  Synchronises the stream.
extern "C" int fgb_kmer_sort_oversized(const void *src, void *dst, long long n, const void *d_plan, unsigned nover,
                                       unsigned ototal, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (nover == 0) return FGB_OK;
  const kmer_plan P(const_cast<void *>(d_plan),n,0);
  std::vector<uint2> over(nover);
  CUDA_TRY(cudaMemcpyAsync(over.data(),P.over,sizeof(uint2)*nover,cudaMemcpyDeviceToHost,st));
  CUDA_TRY(fgb_stream_wait(st));
  std::sort(over.begin(),over.end(),[](const uint2 &x, const uint2 &y) { return x.x < y.x; });
  //  in bin order, the sorted compact array holds bin k's records at opre[k]
  const int nseg = (int) nover;
  std::vector<unsigned> ofrom(nseg), opre(nseg + 1);
  opre[0] = 0;
  for (int k = 0; k < nseg; k++) { ofrom[k] = over[k].x; opre[k+1] = opre[k] + over[k].y; }
  if (opre[nseg] != ototal) return FGB_ERR_ARG;
  dblock<rec128> d_c1, d_c2; dblock<unsigned char> d_ctmp; dblock<unsigned> d_seg;
  long long ctb = fgb_sort128_tmp_bytes(ototal);
  CUDA_TRY(d_c1.alloc((size_t) ototal+1,st));
  CUDA_TRY(d_c2.alloc((size_t) ototal+1,st));
  CUDA_TRY(d_ctmp.alloc(ctb,st));
  CUDA_TRY(d_seg.alloc(3*(size_t) nseg+1,st));
  CUDA_TRY(cudaMemcpyAsync(d_seg,ofrom.data(),sizeof(unsigned)*nseg,cudaMemcpyHostToDevice,st));
  CUDA_TRY(cudaMemcpyAsync(d_seg+nseg,opre.data(),sizeof(unsigned)*nseg,cudaMemcpyHostToDevice,st));
  CUDA_TRY(cudaMemcpyAsync(d_seg+2*nseg,opre.data(),sizeof(unsigned)*(nseg+1),cudaMemcpyHostToDevice,st));
  int nb = (int) ((ototal + 255) / 256); if (nb > 4736) nb = 4736;
  kmer_copy_segments_kernel<<<nb,256,0,st>>>((const rec128 *) src,d_c1,d_seg,d_seg+nseg,d_seg+2*nseg,nseg,ototal);
  int cinb = 0;
  int rc = fgb_sort128_device(d_c1,d_c2,ototal,0,16,d_ctmp,ctb,&cinb,st);
  if (rc) return rc;
  kmer_copy_segments_kernel<<<nb,256,0,st>>>(cinb ? d_c2 : d_c1,(rec128 *) dst,d_seg+nseg,d_seg,d_seg+2*nseg,nseg,ototal);
  fgb_count_launch(2);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(fgb_stream_wait(st));                      // the staging vectors above must outlive the copies
  return FGB_OK;
}

/***********************************************************************************************
 *  Generic exclusive scan of a u32 array (reduce / scan-of-sums / downsweep), used for stream
 *  compaction of syncmer posts, seeds and work lists.
 **********************************************************************************************/

#define SCAN_THREADS 1024
#define SCAN_ITEMS   8
#define SCAN_TILE    (SCAN_THREADS*SCAN_ITEMS)

__global__ void __launch_bounds__(SCAN_THREADS)
scan_reduce_kernel(const unsigned *__restrict__ data, long long n, unsigned long long *__restrict__ sums)
{ __shared__ unsigned long long ws[32];
  long long t0 = (long long) blockIdx.x * SCAN_TILE;
  unsigned long long s = 0;
  for (int i = 0; i < SCAN_ITEMS; i++)
    { long long idx = t0 + i*SCAN_THREADS + threadIdx.x;
      if (idx < n) s += data[idx];
    }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu,s,o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32)
    { s = ws[threadIdx.x];
      for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu,s,o);
      if (threadIdx.x == 0) sums[blockIdx.x] = s;
    }
}

__global__ void __launch_bounds__(1024)
scan_sums_kernel(unsigned long long *__restrict__ sums, int nb, unsigned long long *__restrict__ total)
{ __shared__ unsigned long long ws[32];
  __shared__ unsigned long long carry_s;
  int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (tid == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < nb; base += 1024)
    { int i = base + tid;
      unsigned long long v = (i < nb) ? sums[i] : 0, inc = v;
      for (int o = 1; o < 32; o <<= 1)
        { unsigned long long t = __shfl_up_sync(0xffffffffu,inc,o);
          if (lane >= o) inc += t;
        }
      if (lane == 31) ws[w] = inc;
      __syncthreads();
      if (w == 0)
        { unsigned long long s = ws[lane], si = s;
          for (int o = 1; o < 32; o <<= 1)
            { unsigned long long t = __shfl_up_sync(0xffffffffu,si,o);
              if (lane >= o) si += t;
            }
          ws[lane] = si - s;
        }
      __syncthreads();
      unsigned long long ex = carry_s + ws[w] + inc - v;
      if (i < nb) sums[i] = ex;
      __syncthreads();
      if (tid == 1023) carry_s = ex + v;
      __syncthreads();
    }
  if (tid == 0 && total != NULL) *total = carry_s;
}

__global__ void __launch_bounds__(SCAN_THREADS)
scan_down_kernel(unsigned *__restrict__ data, long long n, const unsigned long long *__restrict__ sums)
{ __shared__ unsigned ws[32];
  int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  long long t0 = (long long) blockIdx.x * SCAN_TILE + (long long) tid * SCAN_ITEMS;
  unsigned v[SCAN_ITEMS], s = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++)
    { v[i] = (t0 + i < n) ? data[t0+i] : 0;
      s += v[i];
    }
  unsigned inc = warp_incl_scan(s,lane);
  if (lane == 31) ws[w] = inc;
  __syncthreads();
  if (w == 0)
    { unsigned x = ws[lane];
      unsigned xi = warp_incl_scan(x,lane);
      ws[lane] = xi - x;
    }
  __syncthreads();
  unsigned ex = (unsigned) sums[blockIdx.x] + ws[w] + inc - s;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++)
    { if (t0 + i < n) data[t0+i] = ex;
      ex += v[i];
    }
}

long long fgb_dev_scan_tmp_bytes(long long n)
{ long long nb = (n + SCAN_TILE - 1) / SCAN_TILE;
  if (nb < 1) nb = 1;
  return nb * 8 + 64;
}

//  In-place exclusive scan (values mod 2^32); *d_total (device, may be NULL) gets the 64-bit sum.

int fgb_dev_exclusive_scan_u32(unsigned *d_data, long long n, unsigned long long *d_total,
                               void *d_tmp, long long tmp_bytes, cudaStream_t st)
{ if (n <= 0)
    { if (d_total) CUDA_TRY(cudaMemsetAsync(d_total,0,8,st));
      return FGB_OK;
    }
  if (tmp_bytes < fgb_dev_scan_tmp_bytes(n)) return FGB_ERR_ARG;
  int nb = (int) ((n + SCAN_TILE - 1) / SCAN_TILE);
  unsigned long long *sums = (unsigned long long *) d_tmp;
  scan_reduce_kernel<<<nb,SCAN_THREADS,0,st>>>(d_data,n,sums);
  scan_sums_kernel<<<1,1024,0,st>>>(sums,nb,d_total);
  scan_down_kernel<<<nb,SCAN_THREADS,0,st>>>(d_data,n,sums);
  fgb_count_launch(3);
  CUDA_TRY(cudaGetLastError());
  return FGB_OK;
}
