"""Register-resident lists of the specialised unique-condition kernels (cb_core.h: list_load / list_in_tri / list_mask /
list_set_tri), compiled for the host in both element forms (32-bit string ids, CB_LIST_KEYS64).

The set predicates read one membership mask per list pair, and every element loop stops at a warp-uniform bound (the
longest list among the lanes of the warp).  Over lists of length 0..10, lists holding a number / NaN / -0.0, and absent,
error, string, number and bool operands, this checks that
  * isSubset / hasIntersection from the shared mask give the answers (and the `slow` flags) of the full 8 x 8 compare
    grid, hasIntersection also from the mask of the swapped pair;
  * a wider bound than the lane's own length (another lane of the warp holds a longer list) changes no answer of
    list_in_tri or of the set predicates."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>
#include "cb_core.h"
using namespace cb;

static uint64_t box(uint32_t tag, uint64_t pay) { return ((uint64_t)(CB_V64_BOX_BASE | tag) << 48) | pay; }
static uint64_t str(uint32_t id) { return box(CB_V64_STRING, id); }

// the full compare grid over every cached position: what the set predicates computed before the shared mask
static int grid_set_tri(bool subset, const ListRegs &A, const ListRegs &B, bool &slow) {
    if (A.st == 1 || B.st == 1) return TRI_E;
    if (A.st == 3 || B.st == 3) return TRI_E;
    if (A.st == 2 || B.st == 2) { slow = true; return TRI_E; }
    bool any_hit = false, all_hit = true;
    for (int i = 0; i < CB_LC; i++) {
        bool hit = false;
        for (int j = 0; j < CB_LC; j++) hit |= A.e[i] == B.e[j];
        const bool valid = (uint32_t)i < A.len;
        any_hit |= valid && hit;
        all_hit &= !valid || hit;
    }
    return (subset ? all_hit : any_hit) ? TRI_T : TRI_F;
}
static ListRegs widened(ListRegs L) { L.bound = CB_LC; return L; }

int main() {
    std::vector<uint64_t> heap;
    std::vector<uint64_t> vals = {box(CB_V64_ABSENT, 0), box(CB_V64_ERROR, 0), str(3), str(9), 0x4000000000000000ull /* 2.0 */,
                                  box(CB_V64_BOOL, 1), box(CB_V64_NULL, 0)};
    auto list = [&](const std::vector<uint64_t> &el) {
        const uint64_t off = heap.size();
        heap.push_back(el.size());
        heap.insert(heap.end(), el.begin(), el.end());
        vals.push_back(box(CB_V64_LIST, CB_V64_HEAP_BATCH_BIT | off));
    };
    uint64_t rng = 0x9E3779B97F4A7C15ull;
    auto next = [&]() { rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17; return rng; };
    for (uint32_t len = 0; len <= 10; len++)
        for (int k = 0; k < 4; k++) {
            std::vector<uint64_t> el;
            for (uint32_t j = 0; j < len; j++) el.push_back(str(1 + (uint32_t)(next() % 7)));   // small alphabet: hits and repeats
            list(el);
        }
    list({str(1), 0x4000000000000000ull});          // a number element
    list({str(2), CB_V64_CANON_NAN});               // NaN
    list({0x8000000000000000ull, str(3)});          // -0.0
    list({str(4), box(CB_V64_LIST, CB_V64_HEAP_BATCH_BIT)});   // a container element
    BatchView b;
    memset(&b, 0, sizeof b);
    b.heap = heap.data();
    b.heap_words = heap.size();
    TableLayout lay;
    memset(&lay, 0, sizeof lay);
    TableView t;
    t.base = nullptr;
    t.L = &lay;
    std::vector<ListRegs> L;
    for (uint64_t v : vals) L.push_back(list_load(t, b, v));
    long bad = 0, n = 0, n_dec = 0, n_slow = 0;
    for (size_t a = 0; a < vals.size(); a++) {
        const ListRegs &A = L[a];
        const uint32_t own = A.st == 0 || A.st == 2 ? (A.len < CB_LC ? A.len : CB_LC) : 0;
        if (A.bound != own) { printf("bound %zu: %u != %u\n", a, A.bound, own); bad++; }
        for (size_t c = 0; c < vals.size(); c++) {   // x in A
            bool s1 = false, s2 = false;
            const int r1 = list_in_tri(vals[c], A, s1), r2 = list_in_tri(vals[c], widened(A), s2);
            n++;
            if (r1 != r2 || s1 != s2) { printf("in %zu %zu: %d/%d %d/%d\n", c, a, r1, r2, s1, s2); bad++; }
        }
        for (size_t c = 0; c < vals.size(); c++) {
            const ListRegs &B = L[c];
            const uint32_t m = list_mask(A, B), mr = list_mask(B, A), mw = list_mask(widened(A), widened(B));
            for (int subset = 0; subset < 2; subset++) {
                bool sg = false, sm = false, sw = false;
                const int g = grid_set_tri(subset, A, B, sg);
                const int r = list_set_tri(subset, A, B, m, sm);
                const int w = list_set_tri(subset, widened(A), widened(B), mw, sw);
                n++;
                n_dec += g != TRI_E;
                n_slow += sg;
                if (g != r || sg != sm || g != w || sg != sw) { printf("set%d %zu %zu: %d %d %d\n", subset, a, c, g, r, w); bad++; }
                if (!subset) {
                    bool ss = false;
                    const int q = list_set_tri(false, B, A, mr, ss);   // hasIntersection(A, B) from the mask of (B, A)
                    if (q != g || ss != sg) { printf("swapped %zu %zu: %d %d\n", a, c, g, q); bad++; }
                }
            }
        }
    }
    printf("checked %ld decided %ld slow %ld mismatches %ld\n", n, n_dec, n_slow, bad);
    return bad != 0;
}
"""


@pytest.mark.parametrize("form", ["keys32", "keys64"])
def test_list_mask_and_bounds_match_full_grid(form, tmp_path):
    src = tmp_path / "list_regs.cpp"
    src.write_text(HARNESS)
    exe = tmp_path / "list_regs"
    cmd = ["g++", "-O1", "-std=c++17", f"-I{ROOT}/include", f"-I{ROOT}/cerbos_b200/csrc", "-o", str(exe), str(src)]
    if form == "keys64":
        cmd.insert(1, "-DCB_LIST_KEYS64")
    subprocess.run(cmd, check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    last = r.stdout.strip().splitlines()[-1].split()
    checked, decided, slow = int(last[1]), int(last[3]), int(last[5])
    # every kind of outcome is exercised: decided pairs, pairs sent to the general body, errors
    assert checked > 5000 and decided > 1000 and slow > 100, r.stdout[-400:]
