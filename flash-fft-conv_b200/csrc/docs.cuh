// docs.cuh — packed documents regrouped by length for the long convolution (bffc_docs_gather, bffc_docs_scatter).
//
// Rows (B, H, L) hold several documents each.  A document of length l is convolved in a batch of its own length class
// c = max(128, next_pow2(l)), a (n_c, H, c) tensor that the plan of seqlen 2c convolves member by member (the host
// side, INTEGRATION.md §11).  The class batches of every class lie one after the other in one "gathered" buffer of
// H * positions elements, positions = sum over classes of n_c * c.  An item (DocItem) says where one document sits in
// the rows and in that buffer: element (h, t) of item i is gathered element H * dst + h * cls + t.
//
//   gather:  gathered[H * dst + h * cls + t] = t < length ? x[row * bs + h * L + start + t] : 0      (t < cls)
//   scatter: x[row * bs + h * L + start + t] = gathered[H * dst + h * cls + t]                         (t < length)
//
// Items are sorted by dst and tile the buffer ([dst, dst + cls) of consecutive items touch), so a thread finds the item
// of a gathered element by binary search over dst.  The grid is one-dimensional: each thread owns 8 consecutive
// gathered elements (one 16-byte vector: c >= 128 keeps every class row 16-byte aligned in a 16-byte aligned buffer) at
// a time, grid-stride, with 64-bit indices throughout; nothing is placed in gridDim.y / z, so no shape is limited by
// them.  Up to kMaxTensors tensors share one launch (the item lookup is done once for all of them).  The row side is
// read or written as 16-bit scalars: a document may start at any element.  The elements are copied as 16-bit words, so
// the kernels serve bf16 and fp16 alike.  Items whose fields do not fit the rows (row >= B, start + length > L,
// length > cls) are treated as empty: gather writes zeros, scatter writes nothing.
#pragma once
#include <cstdint>

namespace bffc {
namespace docs {

constexpr int kThreads = 256;
constexpr int kVec = 8;                 // 16-bit elements per thread and step: one 16-byte vector of the class batch
constexpr int kMaxTensors = 4;

// one item of the device table (24 bytes; the table is 8-byte aligned)
struct DocItem {
  int32_t row;          // batch row b
  int32_t start;        // first position of the document in its row
  int32_t length;       // l >= 1
  int32_t cls;          // class length c: max(128, next_pow2(l))
  int64_t dst;          // first position of the item's row of its class batch in the gathered buffer (multiple of 128)
};
static_assert(sizeof(DocItem) == 24, "DocItem layout is part of the C ABI");

struct Params {
  const DocItem* items;
  int n_items;
  long long positions;               // sum of cls over the items
  int B, H, L;
  int nt;                            // tensors in use, 1 .. kMaxTensors
  uint16_t* rows[kMaxTensors];       // row side: (B, H, L), rows contiguous, batch stride bs
  long long bs[kMaxTensors];
  uint16_t* gathered[kMaxTensors];   // H * positions elements, 16-byte aligned
};

// the item holding gathered element e: the last one with H * dst <= e
__device__ __forceinline__ int find_item(const DocItem* it, int n, long long e, long long H) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&it[mid].dst) * H <= e) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// Where gathered vector v lives: the row-side offset of its first element (without the tensor's batch offset) and the
// number of its 8 elements that lie inside the document (0 .. 8).
struct Where {
  long long row_off;     // row * bs is added per tensor
  int row;
  int n;
};

__device__ __forceinline__ Where locate(const Params& p, long long e) {
  const int i = find_item(p.items, p.n_items, e, p.H);
  const int row = __ldg(&p.items[i].row), start = __ldg(&p.items[i].start);
  const int length = __ldg(&p.items[i].length), cls = __ldg(&p.items[i].cls);
  const long long off = e - __ldg(&p.items[i].dst) * p.H;
  Where w{0, 0, 0};
  const bool ok = cls > 0 && row >= 0 && row < p.B && start >= 0 && length >= 0 && length <= cls &&
                  static_cast<long long>(start) + length <= p.L && off >= 0 && off < static_cast<long long>(p.H) * cls;
  if (!ok) return w;
  const long long h = off / cls;
  const int t = static_cast<int>(off - h * cls);
  w.row_off = h * p.L + start + t;
  w.row = row;
  w.n = max(0, min(kVec, length - t));
  return w;
}

__global__ void __launch_bounds__(kThreads) gather_kernel(Params p) {
  const long long nvec = p.positions * p.H / kVec;
  for (long long v = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x; v < nvec;
       v += static_cast<long long>(gridDim.x) * kThreads) {
    const Where w = locate(p, v * kVec);
#pragma unroll
    for (int k = 0; k < kMaxTensors; ++k) {
      if (k >= p.nt) break;
      const uint16_t* src = p.rows[k] + w.row * p.bs[k] + w.row_off;
      uint32_t word[kVec / 2];
#pragma unroll
      for (int j = 0; j < kVec / 2; ++j) {
        const uint32_t lo = 2 * j < w.n ? __ldg(src + 2 * j) : 0u;
        const uint32_t hi = 2 * j + 1 < w.n ? __ldg(src + 2 * j + 1) : 0u;
        word[j] = lo | (hi << 16);
      }
      reinterpret_cast<uint4*>(p.gathered[k])[v] = make_uint4(word[0], word[1], word[2], word[3]);
    }
  }
}

__global__ void __launch_bounds__(kThreads) scatter_kernel(Params p) {
  const long long nvec = p.positions * p.H / kVec;
  for (long long v = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x; v < nvec;
       v += static_cast<long long>(gridDim.x) * kThreads) {
    const Where w = locate(p, v * kVec);
    if (w.n == 0) continue;
#pragma unroll
    for (int k = 0; k < kMaxTensors; ++k) {
      if (k >= p.nt) break;
      const uint4 g = __ldg(reinterpret_cast<const uint4*>(p.gathered[k]) + v);
      const uint32_t word[kVec / 2] = {g.x, g.y, g.z, g.w};
      uint16_t* dst = p.rows[k] + w.row * p.bs[k] + w.row_off;
#pragma unroll
      for (int j = 0; j < kVec; ++j)
        if (j < w.n) dst[j] = static_cast<uint16_t>(word[j / 2] >> (16 * (j % 2)));
    }
  }
}

}  // namespace docs
}  // namespace bffc
