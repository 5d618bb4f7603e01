// Host-only unit test of redisearch_b200/csrc/batch_scratch.h over random region lists: every region is 256-byte aligned and
// non-null, no two regions overlap, zero-count regions are null and take no space, and the binding pass ends exactly where the
// sizing pass said it would.
#include "../../redisearch_b200/csrc/batch_scratch.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

using rsb200::BatchScratch;

struct Region {
    size_t elem; // element size in bytes: 1, 4 or 8
    size_t count;
};

static void *take(BatchScratch &s, const Region &r) {
    switch (r.elem) {
    case 1: return s.take<uint8_t>(r.count);
    case 4: return s.take<float>(r.count);
    default: return s.take<uint64_t>(r.count);
    }
}

// the regions of `rs` over `base`; returns the carver's bytes()
static size_t run(const std::vector<Region> &rs, void *base, std::vector<uint8_t *> &ptrs) {
    BatchScratch s(base);
    ptrs.clear();
    for (const Region &r : rs) ptrs.push_back(static_cast<uint8_t *>(take(s, r)));
    if (s.words() != (s.bytes() + 7) / 8) std::exit(10);
    return s.bytes();
}

int main() {
    std::mt19937_64 rng(12345);
    int failures = 0;
    const auto fail = [&](int trial, const char *what) {
        if (failures++ < 10) std::printf("trial %d: %s\n", trial, what);
    };
    for (int trial = 0; trial < 2000; trial++) {
        std::vector<Region> rs(1 + rng() % 24);
        for (Region &r : rs) {
            const size_t sizes[3] = {1, 4, 8};
            r.elem = sizes[rng() % 3];
            const int kind = (int)(rng() % 4); // zero, tiny, odd-sized, large
            r.count = kind == 0 ? 0 : kind == 1 ? 1 + rng() % 3 : kind == 2 ? 2 * (rng() % 500) + 1 : rng() % 100000;
        }
        std::vector<uint8_t *> ptrs;
        const size_t bytes = run(rs, nullptr, ptrs);
        for (uint8_t *p : ptrs)
            if (p) fail(trial, "the sizing pass returned a pointer");

        // zero-count regions take no space: the list without them sizes the same
        std::vector<Region> nonzero;
        for (const Region &r : rs)
            if (r.count) nonzero.push_back(r);
        std::vector<uint8_t *> unused;
        if (run(nonzero, nullptr, unused) != bytes) fail(trial, "zero-count regions changed the size");

        uint8_t *base = static_cast<uint8_t *>(std::aligned_alloc(BatchScratch::kAlign, (bytes / BatchScratch::kAlign + 1) * BatchScratch::kAlign));
        if (run(rs, base, ptrs) != bytes) fail(trial, "the binding pass ended elsewhere than the sizing pass");
        struct Span {
            uint8_t *begin, *end;
            size_t tag;
        };
        std::vector<Span> spans;
        size_t end_max = 0;
        for (size_t i = 0; i < rs.size(); i++) {
            uint8_t *p = ptrs[i];
            if (rs[i].count == 0) {
                if (p) fail(trial, "a zero-count region is not null");
                continue;
            }
            if (!p) {
                fail(trial, "a region is null");
                continue;
            }
            if ((size_t)(p - base) % BatchScratch::kAlign || reinterpret_cast<uintptr_t>(p) % BatchScratch::kAlign)
                fail(trial, "a region is not 256-byte aligned");
            spans.push_back({p, p + rs[i].elem * rs[i].count, i});
            end_max = std::max(end_max, (size_t)(p + rs[i].elem * rs[i].count - base));
        }
        if (end_max != bytes) fail(trial, "the last region does not end at bytes()");
        std::sort(spans.begin(), spans.end(), [](const Span &a, const Span &b) { return a.begin < b.begin; });
        for (size_t i = 1; i < spans.size(); i++)
            if (spans[i].begin < spans[i - 1].end) fail(trial, "two regions overlap");
        // every region keeps what was written to it after all of them were written
        for (const Span &s : spans) std::memset(s.begin, (int)(s.tag & 0xFF), s.end - s.begin);
        for (const Span &s : spans)
            if (std::count(s.begin, s.end, (uint8_t)(s.tag & 0xFF)) != s.end - s.begin) fail(trial, "a region was overwritten");
        std::free(base);
    }
    if (failures) {
        std::printf("batch_scratch: %d failures\n", failures);
        return 1;
    }
    std::printf("batch_scratch: ok\n");
    return 0;
}
