"""List-header prefetch of the specialised unique-condition kernels (cb_core.h: list_header_pf; cb_kernels.h:
check_uc_body), compiled for the host.

A warp pulls towards L2 the list headers its next chunk will read.  The harness runs the kernel's steps for one warp
(slot words of the next chunk, one address per lane and list slot) over batches of contiguous, reversed and scattered
lists, table-heap lists, absent / error / non-list slots and batch-heap maps, lists at the last words of the heap,
offsets past it, a partial last chunk and a sub-range with first > 0.  It checks that every prefetched address is a
word of the batch heap, that a lane prefetches exactly the header list_load reads first for each batch-heap list of
its request, and that a lane past the batch, a table-heap list or a slot that is not a batch-heap list prefetches
nothing."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <vector>
#include "cb_core.h"
using namespace cb;

static uint64_t box(uint32_t tag, uint64_t pay) { return ((uint64_t)(CB_V64_BOX_BASE | tag) << 48) | pay; }
static uint64_t blist(uint64_t off) { return box(CB_V64_LIST, CB_V64_HEAP_BATCH_BIT | off); }

static uint64_t rng = 0x9E3779B97F4A7C15ull;
static uint64_t next() { rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17; return rng; }

struct Batch {
    std::vector<uint64_t> slots;   // [n_slots][stride]
    std::vector<uint64_t> words;   // heap contents
    uint64_t stride = 0;
};

static long n_checked = 0, n_pf = 0, n_none = 0, n_past = 0, bad = 0;

// One warp's prefetch for chunk c2 (relative to bv.first) of list slots `ls`, as check_uc_body issues it.
static void check_chunk(const char *what, const Batch &B, const uint64_t *heap, uint64_t heap_words, uint64_t first, uint64_t count, uint64_t c2,
                        const std::vector<uint32_t> &ls) {
    BatchView bv;
    memset(&bv, 0, sizeof bv);
    bv.slots = B.slots.data(); bv.stride = B.stride; bv.first = first; bv.count = count;
    bv.heap = heap; bv.heap_words = heap_words;
    n_checked++;
    for (uint32_t v : ls)
        for (uint32_t lane = 0; lane < 32; lane++) {
            const uint64_t i2 = c2 * 32 + lane;
            if (i2 >= bv.count) { n_past++; continue; }   // the kernel issues nothing past the batch
            const uint64_t x = bv.slots[v * bv.stride + bv.first + i2];
            const uint64_t *p = list_header_pf(bv, x);
            // what list_load reads first: the header of a batch-heap list (inside the heap)
            const bool batch_list = v64_tag(x) == CB_V64_LIST && (x & CB_V64_HEAP_BATCH_BIT) && (x & (CB_V64_HEAP_BATCH_BIT - 1)) < bv.heap_words;
            if (!p) { n_none++; if (batch_list) { printf("%s: slot %u lane %u: no prefetch for a batch-heap list\n", what, v, lane); bad++; } continue; }
            n_pf++;
            if (p < bv.heap || p >= bv.heap + bv.heap_words) { printf("%s: slot %u lane %u prefetches outside the heap\n", what, v, lane); bad++; }
            if (!batch_list || p != bv.heap + (x & (CB_V64_HEAP_BATCH_BIT - 1))) { printf("%s: slot %u lane %u prefetches a word list_load does not read first\n", what, v, lane); bad++; }
        }
}

// n requests, two list slots (1 and 3) of lists with `len_max` elements at most, written request after request into
// one heap region per slot; slot 0 a string, slot 2 unused.  `order`: 0 in request order, 1 reversed, 2 scattered
static Batch make(uint64_t n, uint32_t len_max, int order, uint64_t pad_words = 0) {
    Batch B;
    B.stride = n;
    B.slots.assign(4 * n, box(CB_V64_ABSENT, 0));
    B.words.assign(pad_words, 0);
    for (uint32_t v : {1u, 3u}) {
        std::vector<uint64_t> offs(n);
        for (uint64_t k = 0; k < n; k++) {
            const uint64_t r = order == 1 ? n - 1 - k : k;
            const uint32_t len = (uint32_t)(next() % (len_max + 1));
            offs[r] = B.words.size();
            B.words.push_back(len);
            for (uint32_t j = 0; j < len; j++) B.words.push_back(box(CB_V64_STRING, 1 + next() % 50));
            if (order == 2) for (uint32_t g = (uint32_t)(next() % 64); g; g--) B.words.push_back(0);   // gaps: scattered lists
        }
        for (uint64_t k = 0; k < n; k++) B.slots[v * n + k] = blist(offs[k]);
    }
    for (uint64_t k = 0; k < n; k++) B.slots[k] = box(CB_V64_STRING, 7);
    return B;
}

int main() {
    const std::vector<uint32_t> ls = {1u, 3u};
    for (int round = 0; round < 16; round++) {   // fresh random lists each round
        {   // contiguous lists, every chunk; then the same lists in reversed order
            for (int order = 0; order < 2; order++) {
                Batch B = make(256, 8, order);
                const uint64_t *h = B.words.data();
                for (uint64_t c = 0; c < 8; c++) check_chunk(order ? "reversed" : "contiguous", B, h, B.words.size(), 0, 256, c, ls);
            }
        }
        {   // scattered lists
            Batch B = make(128, 10, 2);
            const uint64_t *h = B.words.data();
            for (uint64_t c = 0; c < 4; c++) check_chunk("scattered", B, h, B.words.size(), 0, 128, c, ls);
        }
        {   // lists in the table heap, absent / error / non-list slots, batch-heap maps, offsets at and past the heap's end,
            // mixed with lists
            Batch B = make(64, 8, 0);
            const uint64_t kinds[] = {box(CB_V64_LIST, 5), box(CB_V64_ABSENT, 0), box(CB_V64_ERROR, 0), box(CB_V64_STRING, 3), 0x4000000000000000ull,
                                      box(CB_V64_BOOL, 1), box(CB_V64_MAP, CB_V64_HEAP_BATCH_BIT | 4), blist(B.words.size()), blist(1ull << 46)};
            for (uint64_t k = 0; k < 64; k++)
                if (k % 3 != 1) B.slots[1 * 64 + k] = kinds[next() % 9];
            for (uint64_t k = 0; k < 64; k++) B.slots[3 * 64 + k] = kinds[next() % 9];   // no batch-heap list at all
            const uint64_t *h = B.words.data();
            for (uint64_t c = 0; c < 2; c++) check_chunk("non-lists", B, h, B.words.size(), 0, 64, c, ls);
        }
        {   // the last words of the heap: an empty list in the last word, lists ending exactly at the end
            Batch B = make(32, 3, 0);
            B.words.push_back(2); B.words.push_back(box(CB_V64_STRING, 1)); B.words.push_back(box(CB_V64_STRING, 2));
            B.slots[1 * 32 + 31] = blist(B.words.size() - 3);
            B.words.push_back(0);
            B.slots[3 * 32 + 31] = blist(B.words.size() - 1);
            const uint64_t *h = B.words.data();
            check_chunk("heap end", B, h, B.words.size(), 0, 32, 0, ls);
            // a list whose elements run past the end of the heap
            B.words.push_back(5); B.words.push_back(box(CB_V64_STRING, 1));
            B.slots[1 * 32 + 30] = blist(B.words.size() - 2);
            h = B.words.data();
            check_chunk("cut list", B, h, B.words.size(), 0, 32, 0, ls);
        }
        {   // a partial last chunk, and a chunk past the end
            Batch B = make(100, 8, 0);
            const uint64_t *h = B.words.data();
            for (uint64_t c = 0; c < 5; c++) check_chunk("partial", B, h, B.words.size(), 0, 100, c, ls);
        }
        {   // a sub-range with first > 0 (the pipelined path runs sub-ranges of one batch), ending in a partial chunk
            Batch B = make(300, 8, 0, 3);
            const uint64_t *h = B.words.data();
            for (uint64_t c = 0; c < 6; c++) check_chunk("sub-range", B, h, B.words.size(), 77, 150, c, ls);
        }
    }
    printf("checked %ld prefetched %ld none %ld past %ld mismatches %ld\n", n_checked, n_pf, n_none, n_past, bad);
    return bad != 0;
}
"""


def test_list_header_prefetch_inside_heap(tmp_path):
    src = tmp_path / "heap_prefetch.cpp"
    src.write_text(HARNESS)
    exe = tmp_path / "heap_prefetch"
    subprocess.run(["g++", "-O1", "-std=c++17", f"-I{ROOT}/include", f"-I{ROOT}/cerbos_b200/csrc", "-o", str(exe), str(src)], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    last = r.stdout.strip().splitlines()[-1].split()
    pf, none, past = int(last[3]), int(last[5]), int(last[7])
    # every branch is exercised: batch-heap lists, slots with nothing to fetch, lanes past the batch
    assert pf > 1000 and none > 100 and past > 100, r.stdout[-400:]
