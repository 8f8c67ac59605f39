// carve.h — offset arithmetic of a forward's workspace: plain host code with no CUDA dependency, so the host compiler can build
// and test it (tests/native/carve_check.cpp).  Arena::carve (common.cuh) owns the device memory these offsets point into.
#pragma once
#include <stddef.h>

// One carved buffer: the pointer and how many elements it was carved for.  Converts to T*, so it is passed wherever the pointer
// was; code about to write `count` elements into a buffer shared between stages asks fits(count) first.
template <typename T> struct Buf {
    T* p = nullptr;
    size_t cap = 0;
    operator T*() const { return p; }
    bool fits(size_t count) const { return count <= cap; }
};

// Hands out consecutive buffers from `base`, each starting on a 256-byte boundary; `off` is the total taken so far.  With a null
// base it only measures: every pointer is null and `off` ends at the size the same list of takes needs.
struct Carve {
    char* base;
    size_t off = 0;
    explicit Carve(char* base) : base(base) {}
    // `count` elements of T.  A zero-count take occupies no space and yields a null pointer with capacity 0.
    template <typename T> Buf<T> take(size_t count) {
        Buf<T> b;
        if (base && count) b.p = (T*)(base + off);
        b.cap = count;
        off += (count * sizeof(T) + 255) & ~(size_t)255;
        return b;
    }
};
