// Drop-in replacements for the reference's two extern sort entry points, same signatures and
// in-place semantics on HOST byte records, computed on the device:
//
//   void msd_sort (uint8 *array, int64 nelem, int rsize, int ksize, int64 *part, int beg, int end,
//                  int nthreads);                                   MSDsort.c:404 (built -DLCPs)
//   int  rmsd_sort(uint8 *array, int64 nelem, int rsize, int ksize, int nparts, int64 *part,
//                  int nthreads, Range *range);                     RSDsort.c:292
//
// A maintainer links libfastga_b200.so and `#define msd_sort fgb_msd_sort` /
// `#define rmsd_sort fgb_rmsd_sort` (INTEGRATION.md).  Byte records are widened to 128-bit
// words (panel | key | ...), sorted with the radix sort of sort128.cu and narrowed again.
// Equal keys keep their input order here (the reference's in-place sort leaves them in an
// unspecified order; its consumers do not depend on it).
#include "stages.h"
#include <string.h>

typedef unsigned long long u64;

static __device__ __forceinline__ int panel_of(const long long *__restrict__ poff, int np, long long i)
{ int lo = 0, hi = np-1;                        // last panel with poff <= i
  while (lo < hi)
    { int m = (lo+hi+1) >> 1;
      if (poff[m] <= i) lo = m; else hi = m-1;
    }
  return lo;
}

//  msd: word = panel(16) | key (<= 9 bytes, left aligned in 72 bits) | record index(32)

__global__ void msd_pack_kernel(const unsigned char *__restrict__ arr, long long n, int rsize, int ksize,
                                const long long *__restrict__ poff, int np, rec128 *__restrict__ out)
{ long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned char *r = arr + i*rsize;
  u64 khi = 0; unsigned klo = 0;                // key bytes 1..8 -> khi, byte 9 -> klo
  for (int b = 1; b < ksize && b <= 8; b++) khi |= (u64) r[b] << (8*(8-b));
  if (ksize > 9) klo = r[9];
  unsigned pan = (unsigned) panel_of(poff,np,i);
  rec128 w;
  w.hi = ((u64) pan << 40) | (khi >> 24);       // bits 119..104 panel, 103..64 top 40 key bits
  w.lo = (khi << 40) | ((u64) klo << 32) | (unsigned) i;
  st_rec(out + i,w);
}

static __device__ __forceinline__ int lcp_bytes(u64 ahi, unsigned alo, u64 bhi, unsigned blo, int ksize)
{ //  keys as 9 bytes (hi = bytes 1..8, lo = byte 9); MSDsort.c:121-127: 4*i + LCP_Table[a^b]
  u64 x = ahi ^ bhi;
  if (x)
    { int lead = __clzll(x);                    // bit index from the top of byte 1
      int byte = lead >> 3;                     // 0-based key byte -> record byte byte+1
      if (byte + 1 >= ksize) return 0;
      return ((byte+1) << 2) + ((lead & 7) >> 1);
    }
  if (ksize > 9)
    { unsigned y = (alo ^ blo) & 0xff;
      if (y) return (9 << 2) + ((__clz(y) - 24) >> 1);
    }
  return 0;
}

__global__ void msd_unpack_kernel(const rec128 *__restrict__ srt, long long n, int rsize, int ksize,
                                  const unsigned char *__restrict__ src, unsigned char *__restrict__ dst,
                                  int beg)
{ long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  rec128 w = srt[i];
  const unsigned char *r = src + (long long) (unsigned) w.lo * rsize;
  unsigned char *o = dst + i*rsize;
  for (int b = 1; b < rsize; b++) o[b] = r[b];
  int lcp = 0;
  if (i > 0)
    { rec128 p = srt[i-1];
      int pan = (int) (w.hi >> 40) + beg, ppan = (int) (p.hi >> 40) + beg;
      if (pan != ppan)                          // panel boundary (MSDsort.c:485-506)
        lcp = ((pan & 0x300) == (ppan & 0x300)) ? 1 + ((__clz((pan ^ ppan) & 0xff | 0) - 24) >> 1) : 0;
      else
        { u64 ahi = (p.hi << 24) | (p.lo >> 40), bhi = (w.hi << 24) | (w.lo >> 40);
          lcp = lcp_bytes(ahi,(unsigned) (p.lo >> 32) & 0xff,bhi,(unsigned) (w.lo >> 32) & 0xff,ksize);
        }
    }
  o[0] = (unsigned char) lcp;
}

extern "C" void fgb_msd_sort(unsigned char *array, long long nelem, int rsize, int ksize,
                             long long *part, int beg, int end, int nthreads)
{ (void) nthreads;
  long long asize = nelem*rsize;
  if (nelem <= 0) { array[asize] = 1; return; }
  if (ksize > 10 || rsize > 64 || nelem >= 0xffffffffll || end - beg > 65535)
    { fprintf(stderr,"fastga_b200: fgb_msd_sort: record shape outside the device layout\n"); exit(1); }
  int np = end - beg;
  long long *poff = (long long *) malloc(sizeof(long long)*(np+1));
  poff[0] = 0;
  for (int x = 0; x < np; x++) poff[x+1] = poff[x] + part[beg+x]/rsize;
  cudaStream_t st = 0;
  dblock<unsigned char> d_src, d_dst; dblock<long long> d_poff;
  dblock<rec128> d_a, d_b; dblock<unsigned char> d_tmp;
  long long tmpb = fgb_sort128_tmp_bytes(nelem);
  bool ok = d_src.alloc(asize+16,st) == cudaSuccess &&
            d_dst.alloc(asize+16,st) == cudaSuccess &&
            d_poff.alloc(np+1,st) == cudaSuccess &&
            d_a.alloc(nelem+1,st) == cudaSuccess &&
            d_b.alloc(nelem+1,st) == cudaSuccess &&
            d_tmp.alloc(tmpb,st) == cudaSuccess;
  if (!ok) { fprintf(stderr,"fastga_b200: fgb_msd_sort: out of device memory\n"); exit(1); }
  cudaMemcpyAsync(d_src,array,asize,cudaMemcpyHostToDevice,st);
  cudaMemcpyAsync(d_poff,poff,8*(np+1),cudaMemcpyHostToDevice,st);
  int nb = (int) ((nelem + 255) / 256), inb = 0;
  msd_pack_kernel<<<nb,256,0,st>>>(d_src,nelem,rsize,ksize,d_poff,np,d_a);
  //  key = panel (bytes 13,14) + 9 key bytes (4..12): LSD over bytes 4..14
  if (fgb_sort128_device(d_a,d_b,nelem,4,15,d_tmp,tmpb,&inb,st) != FGB_OK)
    { fprintf(stderr,"fastga_b200: fgb_msd_sort: device sort failed\n"); exit(1); }
  msd_unpack_kernel<<<nb,256,0,st>>>(inb ? d_b : d_a,nelem,rsize,ksize,d_src,d_dst,beg);
  cudaMemcpyAsync(array,d_dst,asize,cudaMemcpyDeviceToHost,st);
  if (cudaStreamSynchronize(st) != cudaSuccess)
    { fprintf(stderr,"fastga_b200: fgb_msd_sort: %s\n",cudaGetErrorString(cudaGetLastError())); exit(1); }
  //  first records of the panels are set by the boundary rule; the very first is 0 (MSDsort.c:485)
  array[0] = 0;
  array[asize] = 1;
  free(poff);
}

//  rmsd: the whole record is the key, last byte most significant (RSDsort.c:54-65, :306);
//  word = panel(16) | record bytes reversed (<= 14 bytes)

__global__ void rmsd_pack_kernel(const unsigned char *__restrict__ arr, long long n, int rsize,
                                 const long long *__restrict__ poff, int np, rec128 *__restrict__ out)
{ long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned char *r = arr + i*rsize;
  rec128 w; w.lo = 0; w.hi = 0;
  for (int b = 0; b < rsize; b++)              // byte b of the record -> byte b of the word
    { if (b < 8) w.lo |= (u64) r[b] << (8*b);
      else       w.hi |= (u64) r[b] << (8*(b-8));
    }
  w.hi |= (u64) (unsigned) panel_of(poff,np,i) << 48;
  st_rec(out + i,w);
}

__global__ void rmsd_unpack_kernel(const rec128 *__restrict__ srt, long long n, int rsize,
                                   unsigned char *__restrict__ dst)
{ long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  rec128 w = srt[i];
  unsigned char *o = dst + i*rsize;
  for (int b = 0; b < rsize; b++)
    o[b] = (unsigned char) ((b < 8) ? (w.lo >> (8*b)) : (w.hi >> (8*(b-8))));
}

extern "C" int fgb_rmsd_sort(unsigned char *array, long long nelem, int rsize, int ksize, int nparts,
                             long long *part, int nthreads, fgb_range *parms)
{ long long asize = nelem*rsize;
  if (rsize > 14 || ksize != rsize || nparts > 65535 || nelem >= 0xffffffffll)
    { fprintf(stderr,"fastga_b200: fgb_rmsd_sort: record shape outside the device layout\n"); exit(1); }

  //  thread ranges exactly as RSDsort.c:320-345 (the caller walks them in search_seeds)
  int n = 0, x, beg;
  long long thr = asize / nthreads, off = 0, sum = 0;
  for (x = 0; x < nparts; x++) if (part[x] > 0) break;
  beg = x;
  for (; x < nparts; x++)
    if (part[x] > 0)
      { sum += part[x];
        if (sum >= thr)
          { parms[n].end = x+1; parms[n].beg = beg; parms[n].off = off;
            n += 1;
            thr = (asize * (n+1))/nthreads;
            beg = x+1;
            off = sum;
          }
      }
  if (n > 0 && n < nthreads)
    { parms[n].beg = parms[n].end = parms[n-1].end; parms[n].off = asize; }
  if (nelem <= 1) return n;

  long long *poff = (long long *) malloc(sizeof(long long)*(nparts+1));
  poff[0] = 0;
  for (x = 0; x < nparts; x++) poff[x+1] = poff[x] + part[x]/rsize;
  cudaStream_t st = 0;
  dblock<unsigned char> d_src; dblock<long long> d_poff;
  dblock<rec128> d_a, d_b; dblock<unsigned char> d_tmp;
  long long tmpb = fgb_sort128_tmp_bytes(nelem);
  bool ok = d_src.alloc(asize+16,st) == cudaSuccess &&
            d_poff.alloc(nparts+1,st) == cudaSuccess &&
            d_a.alloc(nelem+1,st) == cudaSuccess &&
            d_b.alloc(nelem+1,st) == cudaSuccess &&
            d_tmp.alloc(tmpb,st) == cudaSuccess;
  if (!ok) { fprintf(stderr,"fastga_b200: fgb_rmsd_sort: out of device memory\n"); exit(1); }
  cudaMemcpyAsync(d_src,array,asize,cudaMemcpyHostToDevice,st);
  cudaMemcpyAsync(d_poff,poff,8*(nparts+1),cudaMemcpyHostToDevice,st);
  int nb = (int) ((nelem + 255) / 256), inb = 0;
  rmsd_pack_kernel<<<nb,256,0,st>>>(d_src,nelem,rsize,d_poff,nparts,d_a);
  //  LSD: record bytes 0..rsize-1 first, then the panel bytes 14,15 (stable passes)
  int inb2 = 0;
  if (fgb_sort128_device(d_a,d_b,nelem,0,rsize,d_tmp,tmpb,&inb,st) != FGB_OK ||
      fgb_sort128_device(inb ? d_b : d_a,inb ? d_a : d_b,nelem,14,16,d_tmp,tmpb,&inb2,st) != FGB_OK)
    { fprintf(stderr,"fastga_b200: fgb_rmsd_sort: device sort failed\n"); exit(1); }
  inb ^= inb2;
  rmsd_unpack_kernel<<<nb,256,0,st>>>(inb ? d_b : d_a,nelem,rsize,d_src);
  cudaMemcpyAsync(array,d_src,asize,cudaMemcpyDeviceToHost,st);
  if (cudaStreamSynchronize(st) != cudaSuccess)
    { fprintf(stderr,"fastga_b200: fgb_rmsd_sort: %s\n",cudaGetErrorString(cudaGetLastError())); exit(1); }
  free(poff);
  return n;
}
