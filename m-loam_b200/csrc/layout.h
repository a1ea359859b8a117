// layout.h — carving one buffer into 256-byte-aligned typed regions.
#pragma once
#include <cstddef>
#include <cstdint>

namespace mloam {

__host__ __device__ inline size_t align256(size_t bytes) { return (bytes + 255) & ~(size_t)255; }

// Bump allocator over a base address.  A layout is code that takes its regions from a Carve in order: run over a null base it only
// adds up the bytes (`size`), run over the reserved buffer it hands out the typed pointers.  ctx.h carve() does both for a DevBuf.
struct Carve {
  uintptr_t base = 0;
  size_t size = 0;
  Carve() = default;
  explicit Carve(void *b) : base(reinterpret_cast<uintptr_t>(b)) {}
  template <typename T>
  T *take(size_t count) {
    T *p = reinterpret_cast<T *>(base + size);
    size += align256(sizeof(T) * count);
    return p;
  }
};

}  // namespace mloam
