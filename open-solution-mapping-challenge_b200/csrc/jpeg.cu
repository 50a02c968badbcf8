// jpeg.cu — baseline / extended sequential Huffman JPEG decoded on the device, bit-exact to libjpeg-turbo as Pillow
// runs it (islow IDCT, fancy upsampling, JFIF YCbCr -> RGB).  The host (mcb200.jpeg) parses the markers, removes the
// byte stuffing, splits the entropy data at its restart markers and builds the Huffman lookup tables; see
// include/mcb200.h for the table layouts.  Five launches per batch (three for the parallel entropy decode), no
// allocation, no synchronisation.
#include <algorithm>

#include "host_common.h"
#include "../../include/mcb200.h"

namespace mcb {
namespace {

constexpr int kLookahead = 9;
constexpr int kHuffWords = (1 << kLookahead) + 18 + 18 + 256;
constexpr int kMaxcode = 1 << kLookahead, kValoff = kMaxcode + 18, kVals = kValoff + 18;
constexpr int kComp0 = 6, kImageWords = kComp0 + 3 * 10, kSegWords = 5;

__constant__ unsigned char kZigzag[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Bit reader over one segment.  acc holds the next bits MSB-first; bits past the segment's end read as zero but are
// never consumed: `avail` counts the real ones, and consuming more than it is the truncation error.
struct Bits {
  const uint8_t* p;
  int left;           // segment bytes not yet in acc
  unsigned long long acc;
  int avail;          // real bits in acc
  __device__ void fill() {
    while (avail <= 56 && left > 0) {
      acc |= (unsigned long long)__ldg(p++) << (56 - avail);
      avail += 8;
      --left;
    }
  }
  __device__ bool skip(int n) {
    if (n > avail) return false;
    acc <<= n;
    avail -= n;
    return true;
  }
};

// one Huffman symbol; returns -1 (data ends) or -2 (no such code)
__device__ __forceinline__ int huff_decode(Bits& b, const int* t) {
  b.fill();
  const int e = t[(int)(b.acc >> (64 - kLookahead))];
  if (e) return b.skip(e >> 8) ? (e & 0xFF) : -1;
  for (int len = kLookahead + 1; len <= 16; ++len) {
    const int code = (int)(b.acc >> (64 - len));
    if (code <= t[kMaxcode + len]) {
      if (!b.skip(len)) return -1;
      return t[kVals + t[kValoff + len] + code];
    }
  }
  return -2;
}

// s raw bits, sign-extended as T.81 EXTEND; false when the data ends
__device__ __forceinline__ bool receive_extend(Bits& b, int s, int& v) {
  if (s == 0) { v = 0; return true; }
  b.fill();
  if (s > b.avail) return false;
  const int r = (int)(b.acc >> (64 - s));
  b.skip(s);
  v = r < (1 << (s - 1)) ? r - (1 << s) + 1 : r;
  return true;
}

// One whole segment by one thread (DC predictors from 0): blocks zeroed and their non-zero coefficients scattered in
// natural order.  Returns 0 or the first error (1 data ends, 2 no such code, 3 index past 63).
__device__ __forceinline__ int decode_segment(const uint8_t* seg, int bytes, int first, int count,
                                              const int* __restrict__ im, const int* tab, int img,
                                              int16_t* __restrict__ coef) {
  const int ncomp = im[0], mcux = im[1];
  Bits b{seg, bytes, 0ull, 0};
  int pred[3] = {0, 0, 0};
  int err = 0;
  for (int m = first; m < first + count && !err; ++m) {
    const int my = m / mcux, mx = m - my * mcux;
    for (int c = 0; c < ncomp && !err; ++c) {
      const int* cp = im + kComp0 + 10 * c;
      const int ch = cp[0], cv = cp[1], bw = cp[2];
      const int* dc = tab + (cp[7] - img * 8) * kHuffWords;
      const int* ac = tab + (cp[8] - img * 8) * kHuffWords;
      for (int v = 0; v < cv && !err; ++v) {
        for (int h = 0; h < ch && !err; ++h) {
          int16_t* blk = coef + ((long)cp[4] + (long)(my * cv + v) * bw + mx * ch + h) * 64;
          uint4* b4 = reinterpret_cast<uint4*>(blk);
#pragma unroll
          for (int i = 0; i < 8; ++i) b4[i] = make_uint4(0, 0, 0, 0);
          int sym = huff_decode(b, dc), val;
          if (sym < 0) { err = sym == -1 ? 1 : 2; break; }
          if (!receive_extend(b, sym, val)) { err = 1; break; }
          pred[c] += val;
          blk[0] = (int16_t)pred[c];
          for (int k = 1; k < 64;) {
            sym = huff_decode(b, ac);
            if (sym < 0) { err = sym == -1 ? 1 : 2; break; }
            const int r = sym >> 4, sz = sym & 15;
            if (sz) {
              k += r;
              if (k > 63) { err = 3; break; }
              if (!receive_extend(b, sz, val)) { err = 1; break; }
              blk[kZigzag[k]] = (int16_t)val;
              ++k;
            } else if (r == 15) {
              k += 16;
            } else {
              break;
            }
          }
        }
      }
    }
  }
  return err;
}

// One thread per independent segment (an image, or one restart interval of it): DC predictors start at 0, so no
// thread waits on another.  One CTA per image: its Huffman tables are staged in shared memory and its threads take the
// image's segments in turn.  Blocks are zeroed and their non-zero coefficients scattered in natural order.
__global__ void __launch_bounds__(32) jpeg_entropy_kernel(const uint8_t* __restrict__ data, const int* __restrict__ segs,
                                                           const int* __restrict__ images,
                                                           const int* __restrict__ huff, int16_t* __restrict__ coef,
                                                           int* __restrict__ status) {
  __shared__ int tab[8 * kHuffWords];
  const int img = blockIdx.x;
  const int* im = images + (long)img * kImageWords;
  const int seg0 = im[4], nseg = im[5];
  for (int i = threadIdx.x; i < 8 * kHuffWords; i += blockDim.x) tab[i] = __ldg(huff + (long)img * 8 * kHuffWords + i);
  __syncthreads();
  for (int s = seg0 + threadIdx.x; s < seg0 + nseg; s += blockDim.x) {
    const int* sg = segs + (long)s * kSegWords;
    const int err = decode_segment(data + sg[1], sg[2], sg[3], sg[4], im, tab, img, coef);
    if (err) atomicMax(status + img, err);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Parallel entropy decode.  The caller cuts each segment into subsequences of kSubBits unstuffed bits, or leaves it
// whole as one subsequence (mcb200.jpeg does that for short segments).  The decoder state at a subsequence boundary
// is the bit offset of the first symbol (Huffman code plus its extra bits) starting at or after it, with the block
// within the MCU and the zigzag index: packed as
// (p, u << 8 | k).  From a state the decode is fully determined; DC predictors are not part of it, because each
// subsequence sums its DC differences per component and the sums are scanned afterwards.
//   1. jpeg_speculate_kernel, one thread per subsequence: a subsequence's first state is guessed by decoding the
//      previous subsequence from its boundary as if a block started there (Huffman codes resynchronise within a few
//      symbols); the subsequence is then decoded from the guess, recording its exit state, the blocks it starts and its
//      DC sums.  Subsequence 0 of a segment starts from the known state and stops at the segment's last block; a
//      segment of one subsequence is decoded and written here by the serial kernel's loop.
//   2. jpeg_resolve_kernel, one warp per split segment: walks the subsequences in order, 32 at a time, in rounds (see
//      resolve_segment).  A stream that never resynchronises costs about one serial decode here, never a wrong
//      result.  Errors and the segment's last block are only taken from exact decodes.
//   3. jpeg_emit_kernel, one thread per subsequence: decodes again from the exact entry state, first block and DC
//      predictors and scatters the coefficients into blocks zeroed by stage 1 (a block crossing a boundary is written
//      by two threads, its DC by the first).
constexpr int kSubBits = 1024;      // subsequence length in bits (DESIGN.md §4.5 has the measurement behind it)
constexpr int kSubThreads = 128;    // threads of a stage-1 / stage-3 CTA: subsequences of one image
constexpr int kResolveWarps = 4;
constexpr int kWarmRestarts = 8;    // guessing: restarts after an invalid code before the guess is given up
constexpr int kCounterWords = 16, kRecWords = 16;
constexpr int kNoEnd = 0x7FFFFFFF;
constexpr int kDone = -1;           // run(): the segment's last block has been decoded
// record words (workspace int32 [kCounterWords + nsub * kRecWords])
enum { kGp, kGuk, kXp, kXuk, kNs, kDc0, kErr = kDc0 + 3, kEp, kEuk, kEb, kEdc0 };
// counters: guesses that held, guesses corrected, the longest run of consecutive corrections, exact re-decodes of a
// record that ended in an error or at the segment's last block
enum { kCntHeld, kCntCorrected, kCntChain, kCntEnd };

// one image's MCU layout, per block of the MCU (u) and per component
struct Layout {
  int mcux, bpm;
  int bw[3], cv[3], ch[3], blk0[3], dc[3], ac[3];
  unsigned char uc[10], uv[10], uh[10];
};

__device__ void stage_image(const int* __restrict__ im, const int* __restrict__ huff, int img, int* tab, Layout& L) {
  for (int i = threadIdx.x; i < 8 * kHuffWords; i += blockDim.x) tab[i] = __ldg(huff + (long)img * 8 * kHuffWords + i);
  if (threadIdx.x == 0) {
    L.mcux = im[1];
    int u = 0;
    for (int c = 0; c < im[0]; ++c) {
      const int* cp = im + kComp0 + 10 * c;
      L.ch[c] = cp[0];
      L.cv[c] = cp[1];
      L.bw[c] = cp[2];
      L.blk0[c] = cp[4];
      L.dc[c] = (cp[7] - img * 8) * kHuffWords;
      L.ac[c] = (cp[8] - img * 8) * kHuffWords;
      for (int v = 0; v < cp[1]; ++v)
        for (int h = 0; h < cp[0]; ++h, ++u) {
          L.uc[u] = (unsigned char)c;
          L.uv[u] = (unsigned char)v;
          L.uh[u] = (unsigned char)h;
        }
    }
    L.bpm = u;
  }
  __syncthreads();
}

// coefficient block of the segment's b-th block
__device__ __forceinline__ long block_at(const Layout& L, int first, int b) {
  const int q = b / L.bpm, u = b - q * L.bpm, m = first + q, my = m / L.mcux, mx = m - my * L.mcux, c = L.uc[u];
  return L.blk0[c] + (long)(my * L.cv[c] + L.uv[u]) * L.bw[c] + mx * L.ch[c] + L.uh[u];
}

struct Dec {
  Bits b;
  int nbits, u, k;
  __device__ void start(const uint8_t* seg, int bytes, int p, int uk) {
    b = Bits{seg + (p >> 3), bytes - (p >> 3), 0ull, 0};
    b.fill();
    b.skip(p & 7);
    nbits = bytes * 8;
    u = uk >> 8;
    k = uk & 0xFF;
  }
  __device__ __forceinline__ int pos() const { return nbits - (b.left * 8 + b.avail); }
  __device__ __forceinline__ int uk() const { return u << 8 | k; }
};

struct Sums {
  int v0, v1, v2;
  __device__ __forceinline__ void add(int c, int x) {
    if (c == 0) v0 += x; else if (c == 1) v1 += x; else v2 += x;
  }
  __device__ __forceinline__ int get(int c) const { return c == 0 ? v0 : c == 1 ? v1 : v2; }
};

// Decodes symbols while the next one starts before bit `end` (a symbol belongs to the subsequence it starts in).
// Returns 0 on reaching `end`, kDone when `limit` blocks have started and a DC symbol would be next, or the serial
// kernel's error code; `at` is then where the failing symbol starts.  With kWrite, coefficients go to the blocks from
// the segment's block b0 on (b0 - 1 when entering inside a block), DC values as pred + the running sums.
template <bool kWrite>
__device__ int run(Dec& d, int end, int limit, const int* tab, const Layout& L, int& ns, Sums& dcs, int& at,
                   int16_t* __restrict__ coef = nullptr, int first = 0, int b0 = 0, Sums pred = Sums{0, 0, 0}) {
  int16_t* blk = nullptr;
  if (kWrite && d.k) blk = coef + block_at(L, first, b0 - 1) * 64;
  for (;;) {
    const int p = d.pos();
    if (p >= end) return 0;
    at = p;
    const int c = L.uc[d.u];
    int val;
    if (d.k == 0) {
      if (ns >= limit) return kDone;
      const int sym = huff_decode(d.b, tab + L.dc[c]);
      if (sym < 0) return sym == -1 ? 1 : 2;
      if (!receive_extend(d.b, sym, val)) return 1;
      dcs.add(c, val);
      if (kWrite) {
        blk = coef + block_at(L, first, b0 + ns) * 64;
        blk[0] = (int16_t)(pred.get(c) + dcs.get(c));
      }
      ++ns;
      d.k = 1;
    } else {
      const int sym = huff_decode(d.b, tab + L.ac[c]);
      if (sym < 0) return sym == -1 ? 1 : 2;
      const int r = sym >> 4, sz = sym & 15;
      if (sz) {
        d.k += r;
        if (d.k > 63) return 3;
        if (!receive_extend(d.b, sz, val)) return 1;
        if (kWrite) blk[kZigzag[d.k]] = (int16_t)val;
        ++d.k;
      } else if (r == 15) {
        d.k += 16;
      } else {
        d.k = 64;
      }
      if (d.k >= 64) {
        d.k = 0;
        d.u = d.u + 1 == L.bpm ? 0 : d.u + 1;
      }
    }
  }
}

// image's subsequence range [lo, hi) and the segment holding subsequence j (last s with sub_first[s] <= j)
__device__ __forceinline__ int segment_of(const int* __restrict__ sub_first, int seg0, int nseg, int j) {
  int lo = seg0, hi = seg0 + nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(sub_first + mid) <= j) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ int sub_end(int idx, int nsub) { return idx == nsub - 1 ? kNoEnd : (idx + 1) * kSubBits; }

// Stage 1.  Grid (images, chunks of kSubThreads subsequences).  A segment of one subsequence is decoded here exactly
// and written out (its blocks zeroed as they start); for longer segments each thread zeroes a share of the segment's
// blocks for stage 3.  Also zeroes the status words and (first CTA) the counters, so no memset launch is needed.
__global__ void __launch_bounds__(kSubThreads) jpeg_speculate_kernel(
    const uint8_t* __restrict__ data, const int* __restrict__ segs, const int* __restrict__ images,
    const int* __restrict__ huff, const int* __restrict__ sub_first, int* __restrict__ ws, int16_t* __restrict__ coef,
    int* __restrict__ status) {
  __shared__ int tab[8 * kHuffWords];
  __shared__ Layout L;
  const int img = blockIdx.x;
  const int* im = images + (long)img * kImageWords;
  const int seg0 = im[4], nseg = im[5];
  if (blockIdx.y == 0 && threadIdx.x == 0) status[img] = 0;
  if (blockIdx.y == 0 && img == 0 && threadIdx.x < kCounterWords) ws[threadIdx.x] = 0;
  const int lo = __ldg(sub_first + seg0), hi = __ldg(sub_first + seg0 + nseg);
  const int j = lo + blockIdx.y * blockDim.x + threadIdx.x;
  if (lo + (int)(blockIdx.y * blockDim.x) >= hi) return;
  stage_image(im, huff, img, tab, L);
  if (j >= hi) return;
  const int s = segment_of(sub_first, seg0, nseg, j);
  const int idx = j - __ldg(sub_first + s), nsub = __ldg(sub_first + s + 1) - __ldg(sub_first + s);
  const int* sg = segs + (long)s * kSegWords;
  const uint8_t* seg = data + sg[1];
  const int bytes = sg[2], total = sg[4] * L.bpm;
  int* rec = ws + kCounterWords + (long)j * kRecWords;
  Dec d;
  int ns = 0, at = 0, gp = 0, guk = 0, err;
  Sums dcs{0, 0, 0};
  if (nsub == 1) {                    // the whole segment, exactly, as the serial kernel decodes it
    rec[kErr] = decode_segment(seg, bytes, sg[3], sg[4], im, tab, img, coef);
    rec[kEp] = -1;                    // nothing left for stage 3
    return;
  }
  // zero this subsequence's share of the segment's blocks for stage 3, which writes a block from two threads when it
  // crosses a boundary
  for (long b = (long)idx * total / nsub; b < (long)(idx + 1) * total / nsub; ++b) {
    uint4* b4 = reinterpret_cast<uint4*>(coef + block_at(L, sg[3], (int)b) * 64);
#pragma unroll
    for (int i = 0; i < 8; ++i) b4[i] = make_uint4(0, 0, 0, 0);
  }
  if (idx == 0) {
    d.start(seg, bytes, 0, 0);
    err = run<false>(d, sub_end(0, nsub), total, tab, L, ns, dcs, at);
  } else {
    const int boundary = idx * kSubBits;
    int q = boundary - kSubBits;
    gp = -1;
    for (int t = 0; t <= kWarmRestarts && q < boundary; ++t) {
      int wns = 0;
      Sums wdc{0, 0, 0};
      d.start(seg, bytes, q, 0);
      if (run<false>(d, boundary, kNoEnd, tab, L, wns, wdc, at) == 0) {
        gp = d.pos();
        guk = d.uk();
        break;
      }
      q = at + 1;
    }
    err = 0;
    if (gp >= 0) {
      d.start(seg, bytes, gp, guk);
      err = run<false>(d, sub_end(idx, nsub), kNoEnd, tab, L, ns, dcs, at);
    }
  }
  rec[kGp] = gp;
  rec[kGuk] = guk;
  rec[kXp] = d.pos();
  rec[kXuk] = d.uk();
  rec[kNs] = ns;
  rec[kDc0] = dcs.v0;
  rec[kDc0 + 1] = dcs.v1;
  rec[kDc0 + 2] = dcs.v2;
  rec[kErr] = err;
  rec[kEp] = idx == 0 ? 0 : -1;   // exact entry: known for subsequence 0, set by stage 2 for the others
  rec[kEuk] = 0;
  rec[kEb] = 0;
  rec[kEdc0] = rec[kEdc0 + 1] = rec[kEdc0 + 2] = 0;
}

__device__ __forceinline__ int warp_excl_scan(int v, int lane) {
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  return x - v;
}

// Stage 2 for one segment of more than one subsequence, by the whole warp, 32 records at a time.  Each round takes
// the records whose entry equals their predecessor's exit (warp scans give their first block and DC predictors); the
// first record that does not is decoded exactly from its true entry, and in the same round every later record whose
// predecessor's exit moved is decoded again from it, so scattered wrong guesses are corrected side by side and a
// stream that never resynchronises costs one subsequence per round, about serial time.
__device__ __forceinline__ void resolve_segment(const uint8_t* __restrict__ data, const int* __restrict__ segs,
                                                const int* __restrict__ sub_first, int* __restrict__ ws,
                                                int* __restrict__ status, const int* tab, const Layout& L, int img,
                                                int s, int lane) {
  const int* sg = segs + (long)s * kSegWords;
  const uint8_t* seg = data + sg[1];
  const int bytes = sg[2], total = sg[4] * L.bpm;
  const int sub0 = __ldg(sub_first + s), nsub = __ldg(sub_first + s + 1) - sub0;
  int ep = 0, euk = 0, eb = 0, chain = 0, longest = 0, held = 0, corrected = 0, ended = 0;
  Sums pred{0, 0, 0};
  bool alive = true;
  for (int base = 0; base < nsub && alive; base += 32) {
    const int cnt = min(32, nsub - base), idx = base + lane;
    int* rec = ws + kCounterWords + (long)(sub0 + min(idx, nsub - 1)) * kRecWords;
    const int gp = rec[kGp], guk = rec[kGuk];
    int ent = gp, entuk = guk;             // the entry the lane's decode below started from
    int xp = rec[kXp], xuk = rec[kXuk], ns = rec[kNs], er = rec[kErr];
    Sums dc{rec[kDc0], rec[kDc0 + 1], rec[kDc0 + 2]};
    int from = 0;
    while (alive && from < cnt) {
      const bool in = lane >= from && lane < cnt;
      int pp = __shfl_up_sync(0xffffffffu, xp, 1), puk = __shfl_up_sync(0xffffffffu, xuk, 1);
      if (lane == from) {
        pp = ep;
        puk = euk;
      }
      if (in && (pp != ent || puk != entuk) && pp == gp && puk == guk) {
        xp = rec[kXp];                     // the predecessor's exit is back at the stage-1 guess: reuse its decode
        xuk = rec[kXuk];
        ns = rec[kNs];
        er = rec[kErr];
        dc = Sums{rec[kDc0], rec[kDc0 + 1], rec[kDc0 + 2]};
        ent = gp;
        entuk = guk;
      }
      // every lane's (entry, decode) pair is self-consistent; compare against the exits as they now stand
      pp = __shfl_up_sync(0xffffffffu, xp, 1);
      puk = __shfl_up_sync(0xffffffffu, xuk, 1);
      if (lane == from) {
        pp = ep;
        puk = euk;
      }
      const int bl = eb + warp_excl_scan(in ? ns : 0, lane);
      const int p0 = pred.v0 + warp_excl_scan(in ? dc.v0 : 0, lane),
                p1 = pred.v1 + warp_excl_scan(in ? dc.v1 : 0, lane),
                p2 = pred.v2 + warp_excl_scan(in ? dc.v2 : 0, lane);
      const bool ok = in && pp == ent && puk == entuk && er == 0 && bl + ns <= total;
      const unsigned bad = __ballot_sync(0xffffffffu, in && !ok);
      const int f = bad ? __ffs(bad) - 1 : cnt;
      const bool take = lane >= from && lane < f;
      if (take) {
        rec[kEp] = pp;
        rec[kEuk] = puk;
        rec[kEb] = bl;
        rec[kEdc0] = p0;
        rec[kEdc0 + 1] = p1;
        rec[kEdc0 + 2] = p2;
      }
      const unsigned fixed = __ballot_sync(0xffffffffu, take && (ent != gp || entuk != guk));
      for (int l = from; l < f; ++l) {     // counters, in subsequence order
        if (fixed >> l & 1u) {
          ++corrected;
          longest = max(longest, ++chain);
        } else {
          ++held;
          chain = 0;
        }
      }
      if (f > from) {
        const int l = f - 1;
        ep = __shfl_sync(0xffffffffu, xp, l);
        euk = __shfl_sync(0xffffffffu, xuk, l);
        eb = __shfl_sync(0xffffffffu, bl + ns, l);
        pred = Sums{__shfl_sync(0xffffffffu, p0 + dc.v0, l), __shfl_sync(0xffffffffu, p1 + dc.v1, l),
                    __shfl_sync(0xffffffffu, p2 + dc.v2, l)};
      }
      if (f == cnt) break;
      // lane f from its true entry (exactly, to the segment's last block); later lanes from their predecessor's exit
      const bool exact = lane == f;
      if (exact || (lane > f && lane < cnt && (pp != ent || puk != entuk))) {
        const int sp = exact ? ep : pp, suk = exact ? euk : puk;
        if (exact) {
          rec[kEp] = ep;
          rec[kEuk] = euk;
          rec[kEb] = eb;
          rec[kEdc0] = pred.v0;
          rec[kEdc0 + 1] = pred.v1;
          rec[kEdc0 + 2] = pred.v2;
        }
        Dec d;
        int at;
        ns = 0;
        dc = Sums{0, 0, 0};
        d.start(seg, bytes, sp, suk);
        er = run<false>(d, sub_end(idx, nsub), exact ? total - eb : kNoEnd, tab, L, ns, dc, at);
        xp = d.pos();
        xuk = d.uk();
        ent = sp;
        entuk = suk;
      }
      if (__shfl_sync(0xffffffffu, gp != ep || guk != euk, f)) {
        ++corrected;
        longest = max(longest, ++chain);
      } else {
        ++ended;
        chain = 0;
      }
      const int rer = __shfl_sync(0xffffffffu, er, f);
      if (rer > 0 && lane == 0) atomicMax(status + img, rer);
      if (rer != 0) alive = false;
      ep = __shfl_sync(0xffffffffu, xp, f);
      euk = __shfl_sync(0xffffffffu, xuk, f);
      eb += __shfl_sync(0xffffffffu, ns, f);
      pred.v0 += __shfl_sync(0xffffffffu, dc.v0, f);
      pred.v1 += __shfl_sync(0xffffffffu, dc.v1, f);
      pred.v2 += __shfl_sync(0xffffffffu, dc.v2, f);
      from = f + 1;
    }
  }
  if (lane == 0) {
    atomicAdd(ws + kCntHeld, held);
    atomicAdd(ws + kCntCorrected, corrected);
    atomicMax(ws + kCntChain, longest);
    atomicAdd(ws + kCntEnd, ended);
  }
}

// Stage 2.  One CTA per image; each warp takes 32 segments at a time: a one-subsequence segment was decoded exactly by
// stage 1, and the warp resolves the others one after another.
__global__ void __launch_bounds__(32 * kResolveWarps, 1) jpeg_resolve_kernel(
    const uint8_t* __restrict__ data, const int* __restrict__ segs, const int* __restrict__ images,
    const int* __restrict__ huff, const int* __restrict__ sub_first, int* __restrict__ ws, int* __restrict__ status) {
  __shared__ int tab[8 * kHuffWords];
  __shared__ Layout L;
  const int img = blockIdx.x;
  const int* im = images + (long)img * kImageWords;
  const int seg0 = im[4], nseg = im[5];
  stage_image(im, huff, img, tab, L);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int g = warp * 32; g < nseg; g += 32 * kResolveWarps) {
    const int s = seg0 + g + lane;
    const int nsub = g + lane < nseg ? __ldg(sub_first + s + 1) - __ldg(sub_first + s) : 0;
    if (nsub == 1) {
      const int er = ws[kCounterWords + (long)__ldg(sub_first + s) * kRecWords + kErr];
      if (er > 0) atomicMax(status + img, er);
    }
    unsigned multi = __ballot_sync(0xffffffffu, nsub > 1);
    while (multi) {
      const int l = __ffs(multi) - 1;
      multi &= multi - 1;
      resolve_segment(data, segs, sub_first, ws, status, tab, L, img, seg0 + g + l, lane);
    }
  }
}

// Stage 3.  Same grid as stage 1.
__global__ void __launch_bounds__(kSubThreads) jpeg_emit_kernel(
    const uint8_t* __restrict__ data, const int* __restrict__ segs, const int* __restrict__ images,
    const int* __restrict__ huff, const int* __restrict__ sub_first, const int* __restrict__ ws,
    int16_t* __restrict__ coef) {
  __shared__ int tab[8 * kHuffWords];
  __shared__ Layout L;
  const int img = blockIdx.x;
  const int* im = images + (long)img * kImageWords;
  const int seg0 = im[4], nseg = im[5];
  const int lo = __ldg(sub_first + seg0), hi = __ldg(sub_first + seg0 + nseg);
  const int j = lo + blockIdx.y * blockDim.x + threadIdx.x;
  if (lo + (int)(blockIdx.y * blockDim.x) >= hi) return;
  stage_image(im, huff, img, tab, L);
  if (j >= hi) return;
  const int* rec = ws + kCounterWords + (long)j * kRecWords;
  const int ep = rec[kEp];
  if (ep < 0) return;                 // after the segment's last block or its first error, or written by stage 1
  const int s = segment_of(sub_first, seg0, nseg, j);
  const int idx = j - __ldg(sub_first + s), nsub = __ldg(sub_first + s + 1) - __ldg(sub_first + s);
  const int* sg = segs + (long)s * kSegWords;
  const int eb = rec[kEb];
  Dec d;
  d.start(data + sg[1], sg[2], ep, rec[kEuk]);
  int ns = 0, at;
  Sums dcs{0, 0, 0};
  run<true>(d, sub_end(idx, nsub), sg[4] * L.bpm - eb, tab, L, ns, dcs, at, coef, sg[3], eb,
            Sums{rec[kEdc0], rec[kEdc0 + 1], rec[kEdc0 + 2]});
}

// libjpeg's jpeg_idct_islow constants (CONST_BITS 13)
constexpr long long F0_298 = 2446, F0_390 = 3196, F0_541 = 4433, F0_765 = 6270, F0_899 = 7373, F1_175 = 9633,
                    F1_501 = 12299, F1_847 = 15137, F1_961 = 16069, F2_053 = 16819, F2_562 = 20995, F3_072 = 25172;
constexpr int kConstBits = 13, kPass1Bits = 2;

// one 1-D islow pass on in[0..7] (stride-free), results before descaling in out[0..7]
__device__ __forceinline__ void idct_1d(const long long* in, long long* out) {
  long long z2 = in[2], z3 = in[6];
  long long z1 = (z2 + z3) * F0_541;
  long long tmp2 = z1 + z3 * -F1_847;
  long long tmp3 = z1 + z2 * F0_765;
  z2 = in[0];
  z3 = in[4];
  long long tmp0 = (z2 + z3) * (1LL << kConstBits);
  long long tmp1 = (z2 - z3) * (1LL << kConstBits);
  const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = in[7];
  tmp1 = in[5];
  tmp2 = in[3];
  tmp3 = in[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * F1_175;
  tmp0 *= F0_298;
  tmp1 *= F2_053;
  tmp2 *= F3_072;
  tmp3 *= F1_501;
  z1 *= -F0_899;
  z2 *= -F2_562;
  z3 = z3 * -F1_961 + z5;
  z4 = z4 * -F0_390 + z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  out[0] = tmp10 + tmp3;
  out[7] = tmp10 - tmp3;
  out[1] = tmp11 + tmp2;
  out[6] = tmp11 - tmp2;
  out[2] = tmp12 + tmp1;
  out[5] = tmp12 - tmp1;
  out[3] = tmp13 + tmp0;
  out[4] = tmp13 - tmp0;
}

__device__ __forceinline__ long long descale(long long x, int n) { return (x + (1LL << (n - 1))) >> n; }

// the sample limit as Pillow's libjpeg-turbo applies it on x86: its AVX2 islow IDCT packs the descaled result with
// signed saturation and adds 128, so a value outside [-128, 127] saturates (the C code's range-limit table would wrap
// values beyond +-512; the two agree inside that)
__device__ __forceinline__ uint8_t range_limit(int x) { return (uint8_t)(min(max(x, -128), 127) + 128); }

// One thread per 8x8 block: dequantise (the table entry as libjpeg's 16-bit multiplier), columns, int32 workspace,
// rows, saturation to the sample range.  Blocks of one image are contiguous from its first component's offset.
__global__ void __launch_bounds__(128) jpeg_idct_kernel(const int16_t* __restrict__ coef, const int* __restrict__ qt,
                                                         const int* __restrict__ images, int n, int n_blocks,
                                                         uint8_t* __restrict__ planes) {
  const int blk = blockIdx.x * blockDim.x + threadIdx.x;
  if (blk >= n_blocks) return;
  int lo = 0, hi = n - 1;                         // last image whose first block <= blk
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(images + (long)mid * kImageWords + kComp0 + 4) <= blk) lo = mid; else hi = mid - 1;
  }
  const int* im = images + (long)lo * kImageWords;
  int c = 0;
  for (int k = 1; k < __ldg(im); ++k)
    if (__ldg(im + kComp0 + 4 + 10 * k) <= blk) c = k;
  const int* q = qt + ((long)lo * 3 + c) * 64;
  int16_t x[64];
  const uint4* src = reinterpret_cast<const uint4*>(coef + (long)blk * 64);
#pragma unroll
  for (int i = 0; i < 8; ++i) *reinterpret_cast<uint4*>(x + 8 * i) = __ldg(src + i);
  int ws[64];
#pragma unroll
  for (int col = 0; col < 8; ++col) {
    long long in[8], out[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) in[r] = (long long)((int)x[r * 8 + col] * (int)(int16_t)__ldg(q + r * 8 + col));
    idct_1d(in, out);
#pragma unroll
    for (int r = 0; r < 8; ++r) ws[r * 8 + col] = (int)descale(out[r], kConstBits - kPass1Bits);
  }
  uint32_t packed[16];
#pragma unroll
  for (int row = 0; row < 8; ++row) {
    long long in[8], out[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) in[k] = ws[row * 8 + k];
    idct_1d(in, out);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t w = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        w |= (uint32_t)range_limit((int)descale(out[h * 4 + k], kConstBits + kPass1Bits + 3)) << (8 * k);
      packed[row * 2 + h] = w;
    }
  }
  uint4* dst = reinterpret_cast<uint4*>(planes + (long)blk * 64);
#pragma unroll
  for (int i = 0; i < 4; ++i) dst[i] = make_uint4(packed[4 * i], packed[4 * i + 1], packed[4 * i + 2], packed[4 * i + 3]);
}

// sample (y, x) of a component stored as 8x8 blocks, bw blocks per row
__device__ __forceinline__ int sample(const uint8_t* __restrict__ p, int bw, int y, int x) {
  return __ldg(p + ((long)(y >> 3) * bw + (x >> 3)) * 64 + (y & 7) * 8 + (x & 7));
}

// libjpeg-turbo's upsampled value of one component at output pixel (y, x).  Neighbour samples are clamped into the
// component's downsampled size (jdmainct.c's context rows replicate the first and last rows; jdsample.c's first and
// last columns reduce to the same formula), so padding-block samples are never read.
__device__ __forceinline__ int upsampled(const uint8_t* __restrict__ p, const int* __restrict__ cp, int rx, int ry,
                                         int y, int x) {
  const int bw = cp[2], cw = cp[5], ch = cp[6];
  if (rx == 1 && ry == 1) return sample(p, bw, y, x);
  const int i = ry == 2 ? y >> 1 : y;
  const int j = rx == 2 ? x >> 1 : x;
  if (rx == 2 && cw <= 2) return sample(p, bw, i, j);     // jdsample.c: box filter for a component <= 2 wide
  const int ni = ry == 2 ? min(max((y & 1) ? i + 1 : i - 1, 0), ch - 1) : i;
  if (rx == 1)                                             // h1v2: +1 for the upper output row, +2 for the lower
    return (3 * sample(p, bw, i, j) + sample(p, bw, ni, j) + 1 + (y & 1)) >> 2;
  const int nj = min(max((x & 1) ? j + 1 : j - 1, 0), cw - 1);
  if (ry == 1)                                             // h2v1: +1 even, +2 odd output column
    return (3 * sample(p, bw, i, j) + sample(p, bw, i, nj) + 1 + (x & 1)) >> 2;
  const int s0 = 3 * sample(p, bw, i, j) + sample(p, bw, ni, j);  // h2v2: column sums, then +8 even, +7 odd
  const int s1 = 3 * sample(p, bw, i, nj) + sample(p, bw, ni, nj);
  return (3 * s0 + s1 + 8 - (x & 1)) >> 4;
}

// One thread per output pixel: upsample every component, then jdcolor.c's ycc_rgb_convert with the host-built tables
// (Cr->R, Cb->B, Cr->G, Cb->G at SCALEBITS 16); a grayscale image is replicated to three bands.
__global__ void __launch_bounds__(256) jpeg_upsample_rgb_kernel(const uint8_t* __restrict__ planes,
                                                                 const int* __restrict__ images,
                                                                 const int* __restrict__ tables, int h, int w,
                                                                 uint8_t* __restrict__ out) {
  const int img = blockIdx.y;
  const long pix = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long)h * w) return;
  const int y = (int)(pix / w), x = (int)(pix - (long)y * w);
  const int* gi = images + (long)img * kImageWords;
  const int ncomp = __ldg(gi), hmax = __ldg(gi + 2), vmax = __ldg(gi + 3);
  int v[3] = {0, 0, 0};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (c >= ncomp) break;
    int cp[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) cp[k] = __ldg(gi + kComp0 + 10 * c + k);
    v[c] = upsampled(planes + (long)cp[4] * 64, cp, hmax / cp[0], vmax / cp[1], y, x);
  }
  uint8_t* o = out + ((long)img * h * w + pix) * 3;
  if (ncomp == 1) {
    o[0] = o[1] = o[2] = (uint8_t)v[0];
    return;
  }
  const int yy = v[0], cb = v[1], cr = v[2];
  const int r = yy + __ldg(tables + cr);
  const int g = yy + ((__ldg(tables + 768 + cb) + __ldg(tables + 512 + cr)) >> 16);
  const int b = yy + __ldg(tables + 256 + cb);
  o[0] = (uint8_t)min(max(r, 0), 255);
  o[1] = (uint8_t)min(max(g, 0), 255);
  o[2] = (uint8_t)min(max(b, 0), 255);
}

}  // namespace
}  // namespace mcb

using namespace mcb;
#define ST static_cast<cudaStream_t>(stream)

extern "C" int mcb_jpeg_entropy_decode(const uint8_t* data, const int* segments, int nseg, const int* images,
                                       const int* huff, int n, int16_t* coef, int* status, void* stream) {
  MCB_REQUIRE(data && segments && images && huff && coef && status, "jpeg_entropy_decode: null pointer");
  MCB_REQUIRE(nseg > 0 && n > 0, "jpeg_entropy_decode: %d segments, %d images", nseg, n);
  MCB_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int) * (size_t)n, ST));
  jpeg_entropy_kernel<<<n, 32, 0, ST>>>(data, segments, images, huff, coef, status);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_jpeg_subsequence_bits(void) { return kSubBits; }

extern "C" int mcb_jpeg_entropy_decode_parallel(const uint8_t* data, const int* segments, int nseg, const int* images,
                                                const int* huff, int n, const int* sub_first, int max_image_subs,
                                                int* workspace, int16_t* coef, int* status, void* stream) {
  MCB_REQUIRE(data && segments && images && huff && sub_first && workspace && coef && status,
              "jpeg_entropy_decode_parallel: null pointer");
  MCB_REQUIRE(nseg > 0 && n > 0 && max_image_subs > 0 && max_image_subs <= 65535 * kSubThreads,
              "jpeg_entropy_decode_parallel: %d segments, %d images, %d subsequences", nseg, n, max_image_subs);
  const dim3 grid((unsigned)n, (unsigned)((max_image_subs + kSubThreads - 1) / kSubThreads));
  jpeg_speculate_kernel<<<grid, kSubThreads, 0, ST>>>(data, segments, images, huff, sub_first, workspace, coef, status);
  MCB_LAUNCH_CHECK();
  jpeg_resolve_kernel<<<n, 32 * kResolveWarps, 0, ST>>>(data, segments, images, huff, sub_first, workspace, status);
  MCB_LAUNCH_CHECK();
  jpeg_emit_kernel<<<grid, kSubThreads, 0, ST>>>(data, segments, images, huff, sub_first, workspace, coef);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_jpeg_idct(const int16_t* coef, const int* qt, const int* images, int n, int n_blocks,
                             uint8_t* planes, void* stream) {
  MCB_REQUIRE(coef && qt && images && planes, "jpeg_idct: null pointer");
  MCB_REQUIRE(n > 0 && n_blocks > 0, "jpeg_idct: %d images, %d blocks", n, n_blocks);
  jpeg_idct_kernel<<<(n_blocks + 127) / 128, 128, 0, ST>>>(coef, qt, images, n, n_blocks, planes);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_jpeg_upsample_rgb(const uint8_t* planes, const int* images, const int* tables, int n, int h, int w,
                                     uint8_t* out, void* stream) {
  MCB_REQUIRE(planes && images && tables && out, "jpeg_upsample_rgb: null pointer");
  MCB_REQUIRE(n > 0 && n <= 65535 && h > 0 && w > 0, "jpeg_upsample_rgb: bad shape (n %d, %dx%d)", n, h, w);
  const long hw = (long)h * w;
  jpeg_upsample_rgb_kernel<<<dim3((unsigned)((hw + 255) / 256), n), 256, 0, ST>>>(planes, images, tables, h, w, out);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
