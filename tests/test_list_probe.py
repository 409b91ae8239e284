"""One probe pass per list (cb_core.h: list_probe_key / list_probe / list_in_tri over a hit bit / list_mask), compiled for
the host in both element forms (32-bit string ids, CB_LIST_KEYS64), and the form the generated evaluator gives C3's
list terms (cb_specialize.h: generate_uc).

Over the value families of test_list_regs.py -- lists of length 0..10, lists holding a number / NaN / -0.0 / a container,
absent, error, string, number, bool and null operands -- and with the warp bound at the lane's own length and at CB_LC
(another lane of the warp holds a longer list), this checks that
  * every hit bit of a multi-key probe, read through list_in_tri's status logic, gives the outcome and the `slow` flag
    of a scan of the list's own elements (the compare loop list_in_tri ran before the probes);
  * list_mask and the set predicates over it equal the full 8 x 8 compare grid, `slow` included;
  * a list whose words run past the end of the heap defers, and one that ends on the heap's last word does not."""
import os
import re
import subprocess

import pytest

from hostsim import driver as hostsim

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

// x in L by scanning the list's own elements (no bound, no padding)
static int scan_in_tri(uint64_t x, const ListRegs &L, bool &slow) {
    if (v64_bad(x) || L.st == 1) return TRI_E;
    if (L.st != 0 || v64_tag(x) > CB_V64_STRING || x == CB_V64_CANON_NAN) { slow = true; return TRI_E; }
    bool found = false;
    for (uint32_t j = 0; j < L.len; j++) found |= list_probe_key(x) == L.e[j];
    return found ? TRI_T : TRI_F;
}
static uint32_t grid_mask(const ListRegs &A, const ListRegs &B) {
    uint32_t m = 0;
    for (uint32_t i = 0; i < A.len && i < (uint32_t)CB_LC; i++)
        for (uint32_t j = 0; j < B.len && j < (uint32_t)CB_LC; j++) m |= (uint32_t)(A.e[i] == B.e[j]) << i;
    return m;
}
static int grid_set_tri(bool subset, const ListRegs &A, const ListRegs &B, bool &slow) {
    if (A.st == 1 || B.st == 1) return TRI_E;
    if (A.st == 3 || B.st == 3) return TRI_E;
    if (A.st == 2 || B.st == 2) { slow = true; return TRI_E; }
    const uint32_t m = grid_mask(A, B);
    return (subset ? m == (1u << A.len) - 1u : m != 0u) ? TRI_T : TRI_F;
}
static ListRegs widened(ListRegs L) { L.bound = CB_LC; return L; }

template <int P>
static long probe_all(const std::vector<uint64_t> &vals, const ListRegs &A, size_t a, long &n) {
    long bad = 0;
    for (size_t c0 = 0; c0 < vals.size(); c0 += P) {
        ListKey k[P];
        uint64_t x[P];
        for (int p = 0; p < P; p++) { x[p] = vals[(c0 + p) % vals.size()]; k[p] = list_probe_key(x[p]); }
        const uint32_t h = list_probe(A, k), hw = list_probe(widened(A), k);
        for (int p = 0; p < P; p++) {
            bool s0 = false, s1 = false, s2 = false, s3 = false;
            const int want = scan_in_tri(x[p], A, s0);
            const int r1 = list_in_tri(x[p], A.st, h & (1u << p), s1);
            const int r2 = list_in_tri(x[p], A.st, hw & (1u << p), s2);
            const int r3 = list_in_tri(x[p], A, s3);
            n++;
            if (r1 != want || r2 != want || r3 != want || s1 != s0 || s2 != s0 || s3 != s0) {
                printf("in P=%d x=%zu list=%zu: want %d/%d got %d/%d %d/%d %d/%d\n", P, (c0 + p) % vals.size(), a, want, s0, r1, s1, r2, s2, r3, s3);
                bad++;
            }
        }
    }
    return bad;
}

int main() {
    std::vector<uint64_t> heap;
    std::vector<uint64_t> vals = {box(CB_V64_ABSENT, 0), box(CB_V64_ERROR, 0), str(3), str(9), str(0), 0x4000000000000000ull /* 2.0 */,
                                  0x8000000000000000ull /* -0.0 */, 0ull /* +0.0 */, CB_V64_CANON_NAN, box(CB_V64_BOOL, 1), box(CB_V64_NULL, 0)};
    const size_t n_scalars = vals.size();
    auto list = [&](const std::vector<uint64_t> &el) {
        const uint64_t off = heap.size();
        heap.push_back(el.size());
        heap.insert(heap.end(), el.begin(), el.end());
        vals.push_back(box(CB_V64_LIST, CB_V64_HEAP_BATCH_BIT | off));
    };
    uint64_t rng = 0x2545F4914F6CDD1Dull;
    auto next = [&]() { rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17; return rng; };
    for (uint32_t len = 0; len <= 10; len++)
        for (int k = 0; k < 4; k++) {
            std::vector<uint64_t> el;
            for (uint32_t j = 0; j < len; j++) el.push_back(str((uint32_t)(next() % 8)));   // ids 0..7: hits, misses, repeats
            list(el);
        }
    list({str(1), 0x4000000000000000ull});          // a number element
    list({str(2), CB_V64_CANON_NAN});               // NaN
    list({0x8000000000000000ull, str(3)});          // -0.0
    list({0ull, str(3)});                           // +0.0
    list({str(4), box(CB_V64_LIST, CB_V64_HEAP_BATCH_BIT)});   // a container element
    list({str(5), str(6), str(7)});                 // ends on the heap's last word
    const uint64_t last_list = vals.back();
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
    // the heap's end: the last list is read whole; cut the heap by one word and its last element lies beyond it
    if (L.back().st != 0 || L.back().len != 3) { printf("last list: st %u len %u\n", L.back().st, L.back().len); bad++; }
    b.heap_words = heap.size() - 1;
    const ListRegs cut = list_load(t, b, last_list);
    if (cut.st != 2) { printf("list past the heap's end: st %u\n", cut.st); bad++; }
    b.heap_words = heap.size();
    for (size_t a = 0; a < vals.size(); a++) {
        const ListRegs &A = L[a];
        bad += probe_all<1>(vals, A, a, n);
        bad += probe_all<3>(vals, A, a, n);
        bad += probe_all<8>(vals, A, a, n);
        bad += probe_all<32>(vals, A, a, n);
        for (size_t c = 0; c < vals.size(); c++) {
            const ListRegs &B = L[c];
            const uint32_t mw = list_mask(widened(A), widened(B));
            if (A.st == 0 && B.st == 0 && (list_mask(A, B) != grid_mask(A, B) || mw != grid_mask(A, B))) {
                printf("mask %zu %zu: %x %x want %x\n", a, c, list_mask(A, B), mw, grid_mask(A, B));
                bad++;
            }
            for (int subset = 0; subset < 2; subset++) {
                bool sg = false, sm = false, sw = false;
                const int g = grid_set_tri(subset, A, B, sg);
                const int r = list_set_tri(subset, A, B, list_mask(A, B), sm);
                const int w = list_set_tri(subset, widened(A), widened(B), mw, sw);
                n++;
                n_dec += g != TRI_E;
                n_slow += sg;
                if (g != r || sg != sm || g != w || sg != sw) { printf("set%d %zu %zu: %d %d %d\n", subset, a, c, g, r, w); bad++; }
            }
        }
    }
    (void)n_scalars;
    printf("checked %ld decided %ld slow %ld mismatches %ld\n", n, n_dec, n_slow, bad);
    return bad != 0;
}
"""


@pytest.mark.parametrize("form", ["keys32", "keys64"])
def test_probes_match_scan_and_grid(form, tmp_path):
    src = tmp_path / "list_probe.cpp"
    src.write_text(HARNESS)
    exe = tmp_path / "list_probe"
    cmd = ["g++", "-O1", "-std=c++17", f"-I{ROOT}/include", f"-I{ROOT}/cerbos_b200/csrc", "-o", str(exe), str(src)]
    if form == "keys64":
        cmd.insert(1, "-DCB_LIST_KEYS64")
    subprocess.run(cmd, check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    last = r.stdout.strip().splitlines()[-1].split()
    checked, decided, slow = int(last[1]), int(last[3]), int(last[5])
    assert checked > 20000 and decided > 1000 and slow > 100, r.stdout[-400:]


def test_c3_list_terms_take_the_probe_form():
    """C3's membership terms read hit bits of one probe pass per list, and every list term comes before the first scalar
    term, so that the element registers are dead before the scalar terms run."""
    import workloads as W
    _, ft, _ = W.build(W.C3())
    src = hostsim.generate_uc(ft.blob)[0]
    lines = src[src.index("CB_HD CondWord operator()"):].splitlines()
    terms = [(i, l) for i, l in enumerate(lines) if re.match(r"\s+const int q\d+ = ", l)]
    ins = [l for _, l in terms if "list_in_tri(" in l]
    assert len(ins) == 4
    for l in ins:   # list_in_tri(<probe operand>, cols.l<v>.st, h<v> & <bit>, slow)
        m = re.search(r"list_in_tri\((x(\d+)_\d+), cols\.l(\d+)\.st, h(\d+) & 0x[0-9a-f]+u, slow\)", l)
        assert m and m.group(2) == m.group(3) == m.group(4), l
    probes = [l for l in lines if re.search(r"= list_probe\(cols\.l\d+, k\d+\);", l)]
    assert len(probes) == 2                      # one pass per list slot, P.attr.groups and R.attr.allowed_groups
    assert sum("list_mask(" in l for l in lines) == 1
    list_terms = [i for i, l in terms if "list_in_tri(" in l or "list_set_tri(" in l]
    scalar_terms = [i for i, l in terms if i not in list_terms]
    assert len(list_terms) == 6 and max(list_terms) < min(scalar_terms)
