// bro_concat.cu -- b200_concat_async: the BroCatli splice of many device-resident streams in one stream-ordered pass.
//
// The output equals the host sequence  CreateInstance[WithWindowSize], then per stream NewBrotliFile + ConcatStream over all of
// its bytes, then ConcatFinish  (bro_concat.cuh, the same state machine the host Broccoli ABI runs).  Four launches:
//   k_cat_heads    one thread per stream: is its header sufficient (else the stream is dropped), is the state behind it
//                  determined by its own last two bytes (an "anchor"); the first sufficient stream (atomicMin).
//   k_cat_plan     one thread per stream: starts from the nearest anchor in front of it (almost always the previous stream)
//                  and runs Catli::stream over the streams in between with a discarding sink and over its own with a recording
//                  one.  A stream's output is <= 8 seam bytes (the previous stream's trailing bits, the realigned header, the
//                  look-behind) followed by one byte range of its input.  The first failing stream (atomicMin).
//                  Cost: a stream is an anchor when its header is sufficient, it is longer than 5 bytes and its last two bytes lie
//                  behind its header -- every catable stream of 2 or more input bytes.  Dropped streams (< 4 bytes, e.g. the
//                  1-byte stream of an empty tensor) and the 5-byte stream of 1 input byte are not, and a thread re-runs
//                  Catli::stream over the run of them in front of it: a run of r such streams costs O(r^2) in total and O(r)
//                  dependent steps in its last thread.  Inputs made of long runs of tiny streams are slow, never wrong.
//   k_cat_finish   one block: exclusive scan of the output byte counts, the verdict (first failure, or the first stream that
//                  overflows out_cap), Catli::finish behind the last stream.
//   k_cat_copy     output tiles: seam bytes, and body ranges with aligned 16-byte stores (funnel shifts for the source /
//                  destination misalignment).  Every output byte has one writer; nothing is written unless the verdict is ok.
#include <cuda_runtime.h>

#include <cstdint>

#include "brotli_b200.h"
#include "bro_concat.cuh"

namespace {

using bro::cat::Catli;

constexpr uint8_t kSufficient = 1, kAnchorFirst = 2, kAnchorLater = 4;
constexpr uint32_t kNone = 0xffffffffu;
constexpr int kFinishThreads = 1024, kCopyThreads = 256, kPlanThreads = 128;
constexpr uint64_t kTile = 64 << 10;

struct CatHeader {
  uint32_t first_sufficient;  // atomicMin target: first stream whose header is sufficient
  uint32_t first_error;       // atomicMin target: first stream whose ConcatStream fails
  uint32_t ok;                // verdict of k_cat_finish
  uint32_t pad;
  uint64_t body_total;        // output bytes in front of the finish bytes
  Catli last;                 // the state behind the last stream
};

struct CatPlan {  // what one stream contributes: seam[0, seam_len) then input[body_lo, body_lo + count - seam_len)
  uint64_t body_lo;
  int32_t code;
  uint8_t seam[8];
  uint8_t seam_len;
};

struct Layout {
  CatHeader* H;
  CatPlan* plan;
  uint64_t* count;  // output bytes per stream, then (in place) their exclusive scan
  uint8_t* flags;   // per stream, written by k_cat_heads only
};

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
__host__ __device__ inline Layout layout(void* ws, uint32_t n) {
  uint8_t* p = static_cast<uint8_t*>(ws);
  Layout L;
  L.H = reinterpret_cast<CatHeader*>(p);
  p += align256(sizeof(CatHeader));
  L.plan = reinterpret_cast<CatPlan*>(p);
  p += align256((size_t)n * sizeof(CatPlan));
  L.count = reinterpret_cast<uint64_t*>(p);
  p += align256((size_t)n * sizeof(uint64_t));
  L.flags = p;
  return L;
}

struct NullOut {  // discards, but remembers the last byte (shift_and_check takes it back)
  uint8_t last = 0;
  __device__ size_t avail() const { return ~(size_t)0; }
  __device__ void put(uint8_t b) { last = b; }
  __device__ void copy(const uint8_t*, size_t) {}
  __device__ uint8_t unput() { return last; }
};

struct RecordOut {  // records the seam bytes and the one input range a ConcatStream call with unbounded output writes
  const uint8_t* base;
  uint8_t seam[8];
  int seam_len = 0;
  bool overflow = false;
  uint64_t body_lo = 0, body_len = 0;
  __device__ size_t avail() const { return ~(size_t)0; }
  __device__ void put(uint8_t b) {
    if (seam_len < 8 && body_len == 0) seam[seam_len++] = b;
    else overflow = true;  // cannot happen (bro_concat.cuh: <= 8 puts, all before the copy); reported as 127 if it did
  }
  __device__ void copy(const uint8_t* src, size_t n) {
    if (body_len) overflow = true;
    body_lo = (uint64_t)(src - base);
    body_len = n;
  }
  __device__ uint8_t unput() { return seam[--seam_len]; }
};

__device__ inline int head_bytes(const uint8_t* s, uint64_t n, uint8_t h[bro::cat::kHeaderBytes]) {
  const int nr = n < (uint64_t)bro::cat::kHeaderBytes ? (int)n : bro::cat::kHeaderBytes;
  for (int i = 0; i < bro::cat::kHeaderBytes; ++i) h[i] = i < nr ? s[i] : 0;
  return nr;
}

__global__ void k_cat_heads(const uint8_t* const* streams, const uint64_t* sizes, uint32_t n, Layout L) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint64_t len = sizes[k];
  uint8_t h[bro::cat::kHeaderBytes];
  const int nr = head_bytes(streams[k], len, h);
  uint8_t f = 0;
  if (bro::cat::header_sufficient(h, nr)) {
    f |= kSufficient;
    atomicMin(&L.H->first_sufficient, k);
    // copied as it is (the first stream) or realigned: either way, with more than 5 bytes the state behind the stream is its
    // last two bytes when those lie behind the header (Catli::stream keeps a two-byte look-behind of what it has written)
    if (len > (uint64_t)bro::cat::kHeaderBytes) f |= kAnchorFirst;
    const int varlen = bro::cat::detect_varlen_offset(h, nr);
    if (len > (uint64_t)bro::cat::kHeaderBytes && varlen >= 0 && len - (uint64_t)((varlen + 7) / 8) >= 2) f |= kAnchorLater;
  }
  L.flags[k] = f;
}

__global__ void k_cat_plan(const uint8_t* const* streams, const uint64_t* sizes, uint32_t n, Catli init, Layout L) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t first = init.window_size ? kNone : L.H->first_sufficient;  // the stream copied as it is, if any
  int ws = init.window_size;
  if (first != kNone) {
    uint8_t h[bro::cat::kHeaderBytes];
    head_bytes(streams[first], sizes[first], h);
    int bits;
    if (!bro::cat::parse_window_size(h, &ws, &bits)) ws = 0;  // that stream fails with 125 itself
  }
  // nearest anchor in front of k
  int64_t j = (int64_t)k - 1;
  for (; j >= 0; --j) {
    const uint8_t f = L.flags[j];
    if ((f & kSufficient) && (f & ((uint32_t)j == first ? kAnchorFirst : kAnchorLater))) break;
  }
  Catli st = init;
  bool dead = false;
  if (j >= 0) {
    const uint8_t* s = streams[j];
    const uint64_t len = sizes[j];
    st.init();
    st.window_size = (uint8_t)ws;
    st.last_bytes[0] = s[len - 2];
    st.last_bytes[1] = s[len - 1];
    st.last_bytes_len = 2;
    st.any_bytes_emitted = 1;
  }
  for (int64_t i = j + 1; i < (int64_t)k && !dead; ++i) {
    NullOut o;
    size_t off = 0;
    st.new_brotli_file();
    const int r = st.stream(streams[i], (size_t)sizes[i], &off, o);
    dead = r >= bro::cat::kNotCraftedForAppend || r == bro::cat::kPanic;  // an earlier stream fails: its own thread reports it
  }
  CatPlan p;
  p.body_lo = 0;
  p.code = 0;
  p.seam_len = 0;
  uint64_t cnt = 0;
  if (!dead) {
    RecordOut o;
    o.base = streams[k];
    size_t off = 0;
    st.new_brotli_file();
    int r = st.stream(streams[k], (size_t)sizes[k], &off, o);
    if (r == bro::cat::kPanic || o.overflow) r = bro::cat::kNotCraftedForConcatenation;
    if (r >= bro::cat::kNotCraftedForAppend) {
      p.code = r;
      atomicMin(&L.H->first_error, k);
    } else {
      for (int i = 0; i < o.seam_len; ++i) p.seam[i] = o.seam[i];
      p.seam_len = (uint8_t)o.seam_len;
      p.body_lo = o.body_lo;
      cnt = (uint64_t)o.seam_len + o.body_len;
    }
    if (k + 1 == n) L.H->last = st;
  }
  L.plan[k] = p;
  L.count[k] = cnt;
}

__global__ void __launch_bounds__(kFinishThreads) k_cat_finish(uint32_t n, Catli init, Layout L, uint8_t* out, uint64_t out_cap,
                                                               uint64_t* out_size, int32_t* result) {
  __shared__ uint64_t part[kFinishThreads];
  __shared__ uint32_t overflow_at;
  const uint32_t t = threadIdx.x;
  const uint32_t per = (n + kFinishThreads - 1) / kFinishThreads;
  const uint32_t a = min(n, t * per), b = min(n, a + per);
  uint64_t s = 0;
  for (uint32_t i = a; i < b; ++i) s += L.count[i];
  part[t] = s;
  if (t == 0) overflow_at = kNone;
  __syncthreads();
  for (uint32_t d = 1; d < kFinishThreads; d <<= 1) {  // inclusive Hillis-Steele scan of the per-thread sums
    const uint64_t v = t >= d ? part[t - d] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  uint64_t run = t ? part[t - 1] : 0;
  for (uint32_t i = a; i < b; ++i) {
    const uint64_t c = L.count[i];
    L.count[i] = run;
    if (run + c > out_cap) atomicMin(&overflow_at, i);
    run += c;
  }
  __syncthreads();
  if (t != 0) return;
  const uint64_t body = part[kFinishThreads - 1];
  const uint32_t e = L.H->first_error;
  RecordOut fin;
  fin.base = nullptr;
  if (e == kNone) {  // without a failure the last stream's thread has stored the state behind it
    Catli st = n ? L.H->last : init;
    st.finish(fin);  // unbounded output: always Success, <= 3 bytes
  }
  const uint64_t total = body + (uint64_t)fin.seam_len;
  L.H->body_total = body;
  int32_t code = 0, index = -1;
  if (e != kNone) {
    code = L.plan[e].code;
    index = (int32_t)e;
  } else if (overflow_at != kNone || total > out_cap) {
    code = bro::cat::kNeedsMoreOutput;
    index = overflow_at != kNone ? (int32_t)overflow_at : (int32_t)n;
  }
  L.H->ok = code == 0;
  result[0] = code;
  result[1] = index;
  *out_size = code == 0 ? total : 0;
  if (code == 0)
    for (int i = 0; i < fin.seam_len; ++i) out[body + i] = fin.seam[i];
}

template <int Q>
__device__ inline uint4 shift_bytes(const uint32_t w[8], uint32_t sh) {  // bytes [4Q + sh/8, +16) of w
  uint4 r;
  r.x = __funnelshift_r(w[Q + 0], w[Q + 1], sh);
  r.y = __funnelshift_r(w[Q + 1], w[Q + 2], sh);
  r.z = __funnelshift_r(w[Q + 2], w[Q + 3], sh);
  r.w = __funnelshift_r(w[Q + 3], w[Q + 4], sh);
  return r;
}

// out[b0, b1) = src[0, b1 - b0), by the threads of the block.  Source loads are aligned 16-byte words that each hold at least one
// byte of the range, so they stay inside the pages of the source buffer.
__device__ inline void copy_body(uint8_t* out, uint64_t b0, uint64_t b1, const uint8_t* src) {
  const uintptr_t d0 = reinterpret_cast<uintptr_t>(out + b0), d1 = reinterpret_cast<uintptr_t>(out + b1);
  const uintptr_t w0 = d0 & ~(uintptr_t)15;
  const uint64_t nwords = (d1 - w0 + 15) >> 4;
  const intptr_t delta = reinterpret_cast<intptr_t>(src) - (intptr_t)d0;  // source address = destination address + delta
  const uint32_t r = (uint32_t)((uintptr_t)(w0 + delta) & 15);
  const uint32_t q = r >> 2, sh = (r & 3) * 8;
  for (uint64_t w = threadIdx.x; w < nwords; w += blockDim.x) {
    const uintptr_t A = w0 + (w << 4);
    if (A >= d0 && A + 16 <= d1) {
      const uintptr_t s = A + delta, s0 = s & ~(uintptr_t)15;
      const uint4 x = __ldg(reinterpret_cast<const uint4*>(s0));
      uint4 v;
      if (r == 0) {
        v = x;
      } else {
        const uint4 y = __ldg(reinterpret_cast<const uint4*>(s0 + 16));
        const uint32_t ww[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
        switch (q) {
          case 0: v = shift_bytes<0>(ww, sh); break;
          case 1: v = shift_bytes<1>(ww, sh); break;
          case 2: v = shift_bytes<2>(ww, sh); break;
          default: v = shift_bytes<3>(ww, sh); break;
        }
      }
      *reinterpret_cast<uint4*>(A) = v;
    } else {
      for (uintptr_t p = A > d0 ? A : d0; p < A + 16 && p < d1; ++p)
        *reinterpret_cast<uint8_t*>(p) = *reinterpret_cast<const uint8_t*>(p + delta);
    }
  }
}

__global__ void __launch_bounds__(kCopyThreads) k_cat_copy(const uint8_t* const* streams, const uint64_t* sizes, uint32_t n, Layout L,
                                                           uint8_t* out) {
  if (!L.H->ok) return;
  const uint64_t body = L.H->body_total;
  const uint64_t ntiles = (body + kTile - 1) / kTile;
  __shared__ uint32_t k0;
  for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const uint64_t t0 = t * kTile, t1 = min(t0 + kTile, body);
    if (threadIdx.x == 0) {  // the last stream whose output starts at or before t0
      uint32_t lo = 0, hi = n - 1;
      while (lo < hi) {
        const uint32_t mid = lo + (hi - lo + 1) / 2;
        if (L.count[mid] <= t0) lo = mid;
        else hi = mid - 1;
      }
      k0 = lo;
    }
    __syncthreads();
    const uint32_t first = k0;
    __syncthreads();
    for (uint32_t k = first; k < n; ++k) {
      const uint64_t o = L.count[k];
      if (o >= t1) break;
      const uint64_t end = k + 1 < n ? L.count[k + 1] : body;
      if (end == o) continue;
      const CatPlan& p = L.plan[k];
      const uint32_t sl = p.seam_len;
      if (threadIdx.x < sl) {
        const uint64_t pos = o + threadIdx.x;
        if (pos >= t0 && pos < t1) out[pos] = p.seam[threadIdx.x];
      }
      const uint64_t bs = o + sl;
      const uint64_t b0 = bs > t0 ? bs : t0, b1 = end < t1 ? end : t1;
      if (b0 < b1) copy_body(out, b0, b1, streams[k] + p.body_lo + (b0 - bs));
    }
  }
  (void)sizes;
}

}  // namespace

extern "C" {

size_t b200_concat_workspace_size(uint32_t count) {
  return align256(sizeof(CatHeader)) + align256((size_t)count * sizeof(CatPlan)) + align256((size_t)count * sizeof(uint64_t)) +
         align256(count);
}

int b200_concat_async(const uint8_t* const* d_streams, const uint64_t* d_sizes, uint32_t count, int window_size, uint8_t* out,
                      size_t out_cap, uint64_t* d_out_size, int32_t* d_result, void* d_workspace, size_t workspace_bytes, void* stream) {
  if (!d_out_size || !d_result || !d_workspace || workspace_bytes < b200_concat_workspace_size(count)) return 0;
  if (count && (!d_streams || !d_sizes)) return 0;
  if (count > 0x7fffffffu || window_size < 0 || window_size > 255 || (out_cap && !out)) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Catli init;
  if (!window_size || !init.init_window(window_size)) init.init();  // BroccoliCreateInstanceWithWindowSize (broccoli.rs:60-65)
  const Layout L = layout(d_workspace, count);
  if (cudaMemsetAsync(L.H, 0xff, 2 * sizeof(uint32_t), st) != cudaSuccess) return 0;
  if (count) {
    const uint32_t g = (count + kPlanThreads - 1) / kPlanThreads;
    k_cat_heads<<<g, kPlanThreads, 0, st>>>(d_streams, d_sizes, count, L);
    k_cat_plan<<<g, kPlanThreads, 0, st>>>(d_streams, d_sizes, count, init, L);
  }
  k_cat_finish<<<1, kFinishThreads, 0, st>>>(count, init, L, out, out_cap, d_out_size, d_result);
  if (count) {
    const uint64_t tiles = (out_cap + kTile - 1) / kTile;
    const uint32_t grid = (uint32_t)(tiles < 1 ? 1 : (tiles > 4096 ? 4096 : tiles));
    k_cat_copy<<<grid, kCopyThreads, 0, st>>>(d_streams, d_sizes, count, L, out);
  }
  return cudaGetLastError() == cudaSuccess ? 1 : 0;
}

}  // extern "C"
