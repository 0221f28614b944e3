// lrf_table.cu -- KeySlotSort (lrf_launchers.cuh): the radix sort of the geometry exports' tables, CUB's
// DeviceRadixSort on double buffers, and ExtractScratch, the scratch block of the extracts that sort with it.  The
// only file that includes CUB, so the library carries one copy of its kernels.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>

#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"

namespace lrf {

void KeySlotSort::carve(ScratchCarver& c, long long n) {
  key_buf[0] = c.take<unsigned long long>(n * 8, 256);
  key_buf[1] = c.take<unsigned long long>(n * 8, 256);
  slot_buf[0] = c.take<unsigned int>(n * 4, 256);
  slot_buf[1] = c.take<unsigned int>(n * 4, 256);
  cur = 0;
}

namespace {

// CUB's radix sort of s's pairs by all 64 bits of the key; with a null temp only temp_bytes is computed
cudaError_t radix_sort(KeySlotSort& s, long long n, void* temp, size_t& temp_bytes, cudaStream_t stream) {
  cub::DoubleBuffer<unsigned long long> k(s.key_buf[0], s.key_buf[1]);
  cub::DoubleBuffer<unsigned int> v(s.slot_buf[0], s.slot_buf[1]);
  k.selector = v.selector = s.cur;
  const cudaError_t e = cub::DeviceRadixSort::SortPairs(temp, temp_bytes, k, v, (int)n, 0, 64, stream);
  s.cur = k.selector;
  return e;
}

}  // namespace

cudaError_t KeySlotSort::temp_bytes(long long n, size_t& bytes) {
  KeySlotSort s;
  bytes = 0;
  return radix_sort(s, n, nullptr, bytes, nullptr);
}

cudaError_t KeySlotSort::sort(long long n, void* temp, size_t temp_bytes, cudaStream_t stream) {
  return radix_sort(*this, n, temp, temp_bytes, stream);
}

namespace {

// x's arrays taken from c (null base: only counted): its buffers, then with `temp` the sorts' temporary storage
cudaError_t lay_out(ExtractScratch& x, ScratchCarver& c, bool temp) {
  x.pairs[0].carve(c, x.n);
  if (x.ints) x.index = c.take<int>(x.ints * 4, 256);
  if (x.n2) x.pairs[1].carve(c, x.n2);
  if (!temp) return cudaSuccess;
  cudaError_t e = KeySlotSort::temp_bytes(x.n, x.temp_bytes);
  size_t b = 0;
  if (e == cudaSuccess && x.n2 && (e = KeySlotSort::temp_bytes(x.n2, b)) == cudaSuccess && b > x.temp_bytes)
    x.temp_bytes = b;
  x.temp = c.take(x.temp_bytes, 256);
  return e;
}

}  // namespace

cudaError_t ExtractScratch::bytes(size_t& total, bool temp) const {
  ExtractScratch x = *this;
  ScratchCarver c(nullptr);
  const cudaError_t e = lay_out(x, c, temp);
  total = c.size(256);
  return e;
}

cudaError_t ExtractScratch::carve(void* base) {
  ScratchCarver c(base);
  return lay_out(*this, c, true);
}

}  // namespace lrf
