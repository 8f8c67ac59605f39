// Host check of controlar_b200/csrc/carve.h (the offset arithmetic of a forward's workspace).  For a list of takes it runs the two
// passes Arena::carve runs — measuring on a null base, then assigning on a real one — and checks that the measured total is the
// assigning pass's end offset, that every buffer starts on a 256-byte boundary, that the buffers are disjoint, in order and inside
// the measured total, that a zero-count take is null with capacity 0 and takes no space, and that Buf::fits accepts a write of
// exactly the capacity and refuses one element more.
// usage: carve_check <elem_size>:<count> ...   (elem_size 1, 2 or 4)   -> prints "ok <takes>" or the first violation, exit code 1
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../controlar_b200/csrc/carve.h"

#define FAIL(...) do { printf("FAIL take %zu: ", i); printf(__VA_ARGS__); printf("\n"); return 1; } while (0)

struct Take { int elem; size_t count; };
struct Got { char* p; size_t cap; };

static std::vector<Got> run(Carve& c, const std::vector<Take>& list) {
    std::vector<Got> got;
    for (const Take& t : list) {
        if (t.elem == 1) { Buf<char> b = c.take<char>(t.count); got.push_back({b, b.cap}); }
        else if (t.elem == 2) { Buf<uint16_t> b = c.take<uint16_t>(t.count); got.push_back({(char*)(uint16_t*)b, b.cap}); }
        else { Buf<float> b = c.take<float>(t.count); got.push_back({(char*)(float*)b, b.cap}); }
    }
    return got;
}

int main(int argc, char** argv) {
    std::vector<Take> list;
    for (int a = 1; a < argc; ++a) {
        int elem = 0; unsigned long long count = 0;
        if (sscanf(argv[a], "%d:%llu", &elem, &count) != 2 || (elem != 1 && elem != 2 && elem != 4)) return 2;
        list.push_back({elem, (size_t)count});
    }
    size_t i = 0;
    Carve measure(nullptr);
    for (const Got& g : run(measure, list)) { if (g.p) FAIL("the measuring pass returned a pointer"); ++i; }
    const size_t total = measure.off;
    char* base = (char*)aligned_alloc(256, total + 256);
    Carve c(base);
    const std::vector<Got> got = run(c, list);
    i = list.size();
    if (c.off != total) FAIL("measured %zu bytes, the assigning pass ended at %zu", total, c.off);
    char* cursor = base;                                // end of the previous buffer
    for (i = 0; i < list.size(); ++i) {
        const Got& g = got[i];
        Buf<char> b{g.p, g.cap};
        if (g.cap != list[i].count) FAIL("capacity %zu for a take of %zu", g.cap, list[i].count);
        if (!b.fits(g.cap) || b.fits(g.cap + 1)) FAIL("fits() must accept %zu and refuse %zu", g.cap, g.cap + 1);
        if (list[i].count == 0) { if (g.p) FAIL("a zero-count take must be null"); continue; }
        if (!g.p || ((uintptr_t)g.p & 255)) FAIL("pointer %p is not 256-byte aligned", (void*)g.p);
        if (g.p < cursor) FAIL("overlaps the previous buffer or is out of order");
        if (g.p - cursor >= 256) FAIL("%td bytes of slack in front", g.p - cursor);
        cursor = g.p + g.cap * list[i].elem;
        if (cursor > base + total) FAIL("ends past the measured total");
    }
    free(base);
    printf("ok %zu\n", list.size());
    return 0;
}
