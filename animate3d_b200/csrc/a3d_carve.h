// Bump allocator over a caller-owned workspace or scratch buffer (base may be null for a size query); every piece starts on
// a 256-byte boundary and bytes() rounds the total up to one.
#pragma once
#include <stddef.h>

namespace a3d {

struct Carve {
  char* base;
  size_t off = 0;
  template <class T>
  T* take(size_t count) {
    off = (off + 255) & ~(size_t)255;
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
  size_t bytes() const { return (off + 255) & ~(size_t)255; }
};

}  // namespace a3d
