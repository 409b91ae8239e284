// cb_specialize.h -- host-side generator of table-specialised block evaluators.
//
// The lean kernel body interprets a policy block's records (conditions = lists of 16-byte DNF terms, rows = 16-byte
// records) for every request.  Most of that work is decoding data that is fixed once the table is loaded.  When a
// table is loaded the library therefore emits, for every distinct block SHAPE (same rows + same conditions), a
// function that calls the very same force-inlined device helpers of cb_core.h -- term_tri(), term_lit(),
// row_apply() -- with every record as a compile-time constant, and a `SpecBlocks` dispatcher (switch on the block
// id) that replaces cb::GenericBlocks in the kernels of cb_kernels.h.  NVRTC then folds the switches, operand kinds
// and slot indices away: what is left per term is the operand loads and the compare.  Semantics are identical by
// construction (same helpers, same order), which tests/ check through a host build of the generated text.
//
// Host-only, no CUDA dependencies: tests/hostsim uses it too.
#pragma once
#include <stdint.h>

#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "cerbos_b200_format.h"

namespace cbspec {

struct Limits {
    uint32_t max_shapes = 8;        // more distinct shapes than this: keep the generic walker (code size, NVRTC time:
    uint32_t max_items = 96;        // terms + rows over all shapes     ~1 s for 10 items, ~17 s for 160 on one host core)
};

inline std::string hex(uint32_t v) {
    char buf[16];
    snprintf(buf, sizeof buf, "0x%xu", v);
    return buf;
}
inline std::string hex64(uint64_t v) {
    char buf[32];
    snprintf(buf, sizeof buf, "0x%llxull", (unsigned long long)v);
    return buf;
}

// One DNF term as source text: an expression of type int (TRI_T / TRI_F / TRI_E) that may raise `slow`.
// Shapes with constant operands get the constants as immediates (no table load, no list walk); everything else
// goes through term_tri() with the term words as compile-time constants.
inline std::string term_expr(const uint32_t *w, const uint64_t *consts, const uint64_t *theap) {
    const uint32_t op = w[0] & 0xFFu, flags = (w[0] >> 8) & 0xFFu;
    const std::string sx = "cols.slot(" + std::to_string(w[1]) + "u)";
    switch (op) {
    case CB_TERM_EQ_SC: return "eq_tri(" + sx + ", " + hex64(consts[w[2]]) + ", slow)";
    case CB_TERM_ORD_SC: return "ord_tri(" + hex(flags & CB_TERM_CI_MASK) + ", " + sx + ", " + hex64(consts[w[2]]) + ", slow)";
    case CB_TERM_IN_SC: {
        const uint64_t lst = consts[w[2]];
        const uint64_t *p = theap + (lst & 0xFFFFFFFFFFFFull);
        const uint32_t n = (uint32_t)p[0];
        if (n > 16) break;
        std::string e = "in_const_tri(" + sx + ", slow";
        for (uint32_t j = 0; j < n; j++) e += ", " + hex64(p[1 + j]);
        return e + ")";
    }
    default: break;
    }
    return "term_tri(t, b, cols, pid, U4{" + hex(w[0]) + ", " + hex(w[1]) + ", " + hex(w[2]) + ", " + hex(w[3]) + "}, slow)";
}

// image: host copy of the table image (section offsets in `off`, indexed by CB_SEC_*).  Returns the generated
// source ("" = the table does not qualify: a condition without flat form, too many shapes ...).
inline std::string generate(const uint8_t *image, const uint32_t *off, const uint32_t *meta, const Limits lim = Limits()) {
    const uint32_t n_blocks = meta[CB_META_N_BLOCKS];
    if (n_blocks == 0) return "";
    const uint32_t *blocks = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_BLOCKS]);      // {row_start, n_rows, cond_base, n_conds}
    const uint32_t *rows = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_ROWS]);          // 4 words each
    const uint32_t *conds = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_CONDS]);        // {code_off, code_len, flat_off, flat_info}
    const uint32_t *code = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_CODE]);          // 8-byte instruction slots
    const uint32_t *bs_off = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_BLOCK_SLOTS_OFF]);
    const uint32_t *bs = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_BLOCK_SLOTS]);
    const uint64_t *consts = reinterpret_cast<const uint64_t *>(image + off[CB_SEC_CONSTS_V64]);
    const uint64_t *theap = reinterpret_cast<const uint64_t *>(image + off[CB_SEC_THEAP]);

    std::map<std::vector<uint32_t>, uint32_t> shape_ids;
    std::vector<std::vector<uint32_t>> shape_blocks;     // shape -> block ids
    uint32_t items = 0;
    for (uint32_t bid = 0; bid < n_blocks; bid++) {
        const uint32_t *bl = blocks + 4 * bid;
        if (bl[3] > 31) return "";
        std::vector<uint32_t> key;
        key.push_back(bl[1]);
        key.push_back(bl[3]);
        for (uint32_t r = 0; r < bl[1]; r++) {
            const uint32_t *row = rows + 4 * (bl[0] + r);
            key.push_back(row[0]);            // role | cond << 16
            key.push_back(row[1] & 0xFFFFu);  // drcond
            key.push_back(row[2] & 0xFFu);    // effect
        }
        for (uint32_t c = 0; c < bl[3]; c++) {
            const uint32_t *cd = conds + 4 * (bl[2] + c);
            if (cd[3] == 0 || ((cd[3] >> 16) & 0xFF) != CB_FLAT_DNF) return "";   // no flat form: generic interpreter needed
            key.push_back(cd[2]);
            key.push_back(cd[3]);
        }
        for (uint32_t q = bs_off[bid]; q < bs_off[bid + 1]; q++) key.push_back(bs[q]);
        auto it = shape_ids.find(key);
        if (it == shape_ids.end()) {
            it = shape_ids.emplace(key, (uint32_t)shape_blocks.size()).first;
            shape_blocks.emplace_back();
            items += bl[1];
            for (uint32_t c = 0; c < bl[3]; c++) items += conds[4 * (bl[2] + c) + 3] & 0xFFFFu;
        }
        shape_blocks[it->second].push_back(bid);
    }
    if (shape_blocks.size() > lim.max_shapes || items > lim.max_items) return "";

    std::string s;
    s += "// generated by cb_specialize.h from the loaded table: one straight-line evaluator per block shape\n";
    s += "namespace cb {\n";
    const char *args_decl =
        "const TableView t, const BatchView &b, const Cols &cols, uint32_t pid, uint64_t rp, uint32_t RCP, uint32_t role_all, uint32_t alive, "
        "const uint64_t *ram, uint32_t &D, uint32_t &A, bool &defer";
    for (uint32_t sh = 0; sh < shape_blocks.size(); sh++) {
        const uint32_t bid = shape_blocks[sh][0];
        const uint32_t *bl = blocks + 4 * bid;
        s += "template <typename Cols>\nCB_HD void spec_shape_" + std::to_string(sh) + "(" + args_decl + ") {\n";
        if (bs_off[bid + 1] > bs_off[bid]) {
            s += "    if (!cols.staged()) {";
            for (uint32_t q = bs_off[bid]; q < bs_off[bid + 1]; q++) s += " cols.prefetch_slot(" + std::to_string(bs[q]) + "u);";
            s += " }\n";
        }
        s += "    bool slow = false;\n    uint32_t val = 1u;\n";
        for (uint32_t c = 0; c < bl[3]; c++) {
            const uint32_t *cd = conds + 4 * (bl[2] + c);
            const uint32_t nt = cd[3] & 0xFFFFu, negate = (cd[3] >> 24) & 1u;
            s += "    {   // condition " + std::to_string(c + 1) + "\n        bool any = false, group = true;\n";
            for (uint32_t i = 0; i < nt; i++) {
                const uint32_t *w = code + 2 * (cd[2] + 2 * i);   // a term = two 8-byte instruction slots
                const uint32_t flags = (w[0] >> 8) & 0xFFu;
                s += "        group &= term_lit(" + term_expr(w, consts, theap) + ", " + hex(flags) + ");\n";
                if (flags & CB_TERM_GROUP_END) s += "        any |= group; group = true;\n";
            }
            s += std::string("        val |= (uint32_t)(any != ") + (negate ? "true" : "false") + ") << " + std::to_string(c + 1) + ";\n    }\n";
        }
        s += "    defer |= slow;\n";
        for (uint32_t r = 0; r < bl[1]; r++) {
            const uint32_t *row = rows + 4 * (bl[0] + r);
            s += "    row_apply(ldg(reinterpret_cast<const uint32_t *>(ram + " + std::to_string(r) + ")), U4{" + hex(row[0]) + ", " + hex(row[1] & 0xFFFFu) + ", " +
                 hex(row[2] & 0xFFu) + ", 0u}, rp, RCP, role_all, alive, val, D, A);\n";
        }
        s += "}\n";
    }
    s += "struct SpecBlocks {\n    template <typename Cols>\n    CB_HD void operator()(const TableView t, const BatchView &b, const Cols &cols, uint32_t pid, uint32_t bid, "
         "uint64_t rp, uint32_t RCP, uint32_t role_all, uint32_t alive, const uint64_t *row_am, uint32_t &D, uint32_t &A, bool &defer) const {\n";
    s += "        const uint64_t *ram = row_am + ldg(reinterpret_cast<const uint32_t *>(t.blocks() + bid));   // + row_start\n";
    s += "        switch (bid) {\n";
    for (uint32_t sh = 0; sh < shape_blocks.size(); sh++) {
        s += "       ";
        for (uint32_t bid : shape_blocks[sh]) s += " case " + std::to_string(bid) + ":";
        s += "\n            spec_shape_" + std::to_string(sh) + "(t, b, cols, pid, rp, RCP, role_all, alive, ram, D, A, defer);\n            break;\n";
    }
    s += "        default: defer = true; break;\n        }\n    }\n};\n}  // namespace cb\n";
    return s;
}

// ---- conditions without a flat form: their bytecode programs as straight-line code ------------------------------------
// A condition program (table/bytecode.py: compile_cond) is a condition TREE (all / any / none) over CEL leaf expressions:
//   leaf ... TO_COND [JF_KEEP | JT_KEEP] leaf ... TO_COND (AND | OR) ... [COND_NOT] RET
// A leaf only asks "is the value BOOL true" (errors are plain false: ruletable.go:1467-1486 drops CEL errors), it has no
// side effect, so the tree is a boolean formula over its leaves.  translate_program() splits a program into its leaves
// (ATOMS; the same leaf in several conditions is one atom, evaluated once per request) and the formula; atom_source()
// turns a leaf's instructions into C++ that calls the interpreter's own per-instruction helpers (cb_core.h: op_*,
// do_cmp, do_in ...) with the operand stack as named locals and jumps as gotos -- same helpers, same order, so the
// semantics are the interpreter's by construction; NVRTC then folds constant tags and keeps the stack in registers.
// Programs using instructions outside the supported set (values built in the arena by collecting comprehensions,
// list / map literals, runtime.effectiveDerivedRoles) make the table "not qualify", as before.
struct Ins { uint32_t op, ia, ib, ic; };
struct Atoms {
    std::map<std::vector<uint32_t>, uint32_t> ids;    // normalised instruction list -> atom number
    std::vector<std::string> src;                     // one function per atom
    std::vector<bool> slot_used;
    // per atom: the one slot it reads (CB_NONE32: none or several) and whether it reads anything else of the request
    // (P.id) -- an atom over one slot is a function of that slot's value alone (and of the batch's `now`)
    std::vector<uint32_t> only_slot;
    std::vector<bool> reads_pid;
};

inline bool is_jump(uint32_t op) {
    return op == CB_OP_JF_KEEP || op == CB_OP_JT_KEEP || op == CB_OP_JMP || op == CB_OP_TERN || op == CB_OP_LOOP_INIT || op == CB_OP_LOOP_NEXT || op == CB_OP_LOOP_PRED;
}

// One leaf P[lo, hi) (hi = its TO_COND) -> the body of `template <typename Cols> CB_HD bool uc_atom_K(Ctx &c, const Cols &cols)`.
// "" = an unsupported instruction or a malformed program.
inline std::string atom_source(const std::vector<Ins> &P, uint32_t lo, uint32_t hi, const uint32_t *consts /* cb_const words */, uint32_t n_consts, uint32_t n_slots,
                               std::vector<bool> &slot_used, uint32_t *only_slot = nullptr, bool *reads_pid = nullptr) {
    std::vector<uint32_t> my_slots;
    bool my_pid = false;
    const uint32_t n = hi - lo;
    const int kUnset = -1000;
    std::vector<int> depth(n + 1, kUnset), ldep(n + 1, kUnset);
    std::vector<bool> target(n + 1, false);
    bool bad = false;
    auto set = [&](uint32_t k, int d, int l) {
        if (k > n) { bad = true; return; }
        if (depth[k] == kUnset) { depth[k] = d; ldep[k] = l; }
        else if (depth[k] != d || ldep[k] != l) bad = true;
    };
    auto rel = [&](uint32_t abs) -> uint32_t { if (abs < lo || abs > hi) { bad = true; return 0; } return abs - lo; };
    set(0, 0, 0);
    for (uint32_t k = 0; k < n && !bad; k++) {
        if (depth[k] == kUnset) { bad = true; break; }   // unreachable instruction: not something compile_cond emits
        const Ins &I = P[lo + k];
        const int d = depth[k], l = ldep[k];
        int nd = d;
        bool falls = true;
        switch (I.op) {
        case CB_OP_CONST: case CB_OP_SLOT: case CB_OP_HAS_SLOT: case CB_OP_PID: case CB_OP_NOW: case CB_OP_VAR:
        case CB_OP_CMP_SLOT_CONST: case CB_OP_CMP_SLOT_SLOT: case CB_OP_CMP_SLOT_PID: case CB_OP_IN_SLOT_CONST: case CB_OP_IN_CONST_SLOT:
            nd = d + 1; break;
        case CB_OP_SELECT: case CB_OP_HAS: case CB_OP_NEG: case CB_OP_NOT: case CB_OP_SIZE: case CB_OP_NOERR: case CB_OP_INT: case CB_OP_UINT:
        case CB_OP_DOUBLE: case CB_OP_TIMESTAMP: case CB_OP_DURATION: case CB_OP_DYN: case CB_OP_IN_IP_RANGE: case CB_OP_HIER_SIZE: case CB_OP_TS_GET:
        case CB_OP_MATCHES:
            if (d < 1) bad = true;
            break;
        case CB_OP_INDEX: case CB_OP_EQ: case CB_OP_NE: case CB_OP_LT: case CB_OP_LE: case CB_OP_GT: case CB_OP_GE:
        case CB_OP_ADD: case CB_OP_SUB: case CB_OP_MUL: case CB_OP_DIV: case CB_OP_MOD: case CB_OP_IN:
        case CB_OP_STARTS_WITH: case CB_OP_ENDS_WITH: case CB_OP_CONTAINS: case CB_OP_AND: case CB_OP_OR:
        case CB_OP_HAS_INTERSECTION: case CB_OP_IS_SUBSET: case CB_OP_HIER_REL: case CB_OP_IN_SPLIT:
            if (d < 2) bad = true;
            nd = d - 1; break;
        case CB_OP_HIER_CA: nd = d - (I.ia == 0 ? 1 : 2); if (nd < 1) bad = true; break;
        case CB_OP_FN:   // (format takes its clause record and the list literal's elements: up to a full stack)
            if (I.ib < 1 || I.ib > (I.ia == CB_FN_FORMAT ? (uint32_t)CB_MAX_STACK : 4u) || d < (int)I.ib) bad = true;
            nd = d - ((int)I.ib - 1); break;
        case CB_OP_JF_KEEP: case CB_OP_JT_KEEP: if (d < 1) bad = true; set(rel(I.ic), d, l); target[rel(I.ic)] = true; break;
        case CB_OP_JMP: set(rel(I.ic), d, l); target[rel(I.ic)] = true; falls = false; break;
        case CB_OP_TERN:
            if (d < 1) bad = true;
            nd = d - 1;
            set(rel(I.ic), d - 1, l); target[rel(I.ic)] = true;
            set(rel(I.ib), d, l); target[rel(I.ib)] = true;
            break;
        case CB_OP_LOOP_INIT:
            if (d < 1 || (I.ib & 0xFF) >= CB_LOOP_MAP || l >= CB_MAX_LOOP_DEPTH) bad = true;
            set(rel(I.ic), d, l); target[rel(I.ic)] = true;      // not entered: the comprehension's value is pushed
            set(k + 1, d - 1, l + 1);
            falls = false;
            break;
        case CB_OP_LOOP_NEXT:
            if (d < 1 || (I.ib & 0xFF) >= CB_LOOP_MAP || l < 1) bad = true;
            set(rel(I.ic), d - 1, l); target[rel(I.ic)] = true;  // next element: back to the body
            set(k + 1, d, l - 1);
            falls = false;
            break;
        default: bad = true; break;   // TO_COND / COND_NOT inside a leaf, MKLIST, MKMAP, LOOP_PRED, RUNTIME_EDR, unknown
        }
        if (nd > CB_MAX_STACK) bad = true;
        if (falls && !bad) set(k + 1, nd, l);
    }
    if (bad || depth[n] != 1 || ldep[n] != 0) return "";
    auto S = [](int i) { return "s" + std::to_string(i); };
    auto lab = [](uint32_t k) { return "P" + std::to_string(k); };
    auto cst = [&](uint32_t k) -> std::string {
        if (k >= n_consts) { bad = true; return "mk_err()"; }
        const uint32_t *w = consts + 4 * k;    // {tag, pad, bits lo, bits hi}
        return "mk(" + hex(w[0]) + ", " + hex64((uint64_t)w[2] | (uint64_t)w[3] << 32) + ")";
    };
    auto slot = [&](uint32_t v) -> std::string {
        if (v >= n_slots) { bad = true; return "0ull"; }
        slot_used[v] = true;
        bool seen = false;
        for (uint32_t q : my_slots) seen |= q == v;
        if (!seen) my_slots.push_back(v);
        return "cols.slot(" + std::to_string(v) + "u)";
    };
    int maxd = 1;
    for (uint32_t k = 0; k <= n; k++) if (depth[k] > maxd) maxd = depth[k];
    std::string s = "    Val";
    for (int i = 0; i < maxd; i++) s += std::string(i ? ", " : " ") + S(i);
    s += ";\n    Loop L0, L1; int st_; (void)st_; (void)L0; (void)L1;\n";
    for (uint32_t k = 0; k < n; k++) {
        const Ins &I = P[lo + k];
        const int d = depth[k], l = ldep[k];
        if (target[k]) s += lab(k) + ":;\n";
        const std::string a = S(d - 1), a2 = S(d - 2), top = S(d);   // a: top of stack, a2: below it, top: next free
        s += "    ";
        switch (I.op) {
        case CB_OP_CONST: s += top + " = " + cst(I.ic) + ";"; break;
        case CB_OP_SLOT: s += top + " = decode_v64(" + slot(I.ic) + ", &st_);"; break;
        case CB_OP_HAS_SLOT: s += "decode_v64(" + slot(I.ic) + ", &st_); " + top + " = op_has_slot(st_);"; break;
        case CB_OP_PID: my_pid = true; s += top + " = mk(CB_T_STRING, c.pid);"; break;
        case CB_OP_NOW: s += top + " = mk(CB_T_TS, (uint64_t)c.b->now);"; break;
        case CB_OP_VAR: if (I.ia >= CB_MAX_VARS) bad = true; s += top + " = c.vars[" + std::to_string(I.ia) + "];"; break;
        case CB_OP_SELECT: s += a + " = op_select(c, " + a + ", " + hex(I.ic) + ");"; break;
        case CB_OP_HAS: s += a + " = op_has(c, " + a + ", " + hex(I.ic) + ");"; break;
        case CB_OP_INDEX: s += a2 + " = do_index(c, " + a2 + ", " + a + ");"; break;
        case CB_OP_EQ: case CB_OP_NE: case CB_OP_LT: case CB_OP_LE: case CB_OP_GT: case CB_OP_GE:
            s += a2 + " = do_cmp(c, " + std::to_string(I.op - CB_OP_EQ) + ", " + a2 + ", " + a + ");"; break;
        case CB_OP_ADD: case CB_OP_SUB: case CB_OP_MUL: case CB_OP_DIV: case CB_OP_MOD:
            s += a2 + " = do_arith(c, " + std::to_string(I.op) + ", " + a2 + ", " + a + ");"; break;
        case CB_OP_NEG: s += a + " = op_neg(" + a + ");"; break;
        case CB_OP_NOT: s += a + " = op_not(" + a + ");"; break;
        case CB_OP_IN: s += a2 + " = do_in(c, " + a2 + ", " + a + ");"; break;
        case CB_OP_SIZE: s += a + " = op_size(c, " + a + ");"; break;
        case CB_OP_STARTS_WITH: case CB_OP_ENDS_WITH: case CB_OP_CONTAINS:
            s += a2 + " = do_str2(c, " + std::to_string(I.op) + ", " + a2 + ", " + a + ");"; break;
        case CB_OP_JF_KEEP: s += "if (" + a + ".tag == CB_T_BOOL && " + a + ".u == 0) goto " + lab(I.ic - lo) + ";"; break;
        case CB_OP_JT_KEEP: s += "if (" + a + ".tag == CB_T_BOOL && " + a + ".u == 1) goto " + lab(I.ic - lo) + ";"; break;
        case CB_OP_AND: s += a2 + " = and_or(false, " + a2 + ", " + a + ");"; break;
        case CB_OP_OR: s += a2 + " = and_or(true, " + a2 + ", " + a + ");"; break;
        case CB_OP_JMP: s += "goto " + lab(I.ic - lo) + ";"; break;
        case CB_OP_TERN:
            s += "if (" + a + ".tag == CB_T_BOOL) { if (!" + a + ".u) goto " + lab(I.ic - lo) + "; } else { " + a + " = mk_err(); goto " + lab(I.ib - lo) + "; }";
            break;
        case CB_OP_HAS_INTERSECTION: s += a2 + " = do_set_pred(c, false, " + a2 + ", " + a + ");"; break;
        case CB_OP_IS_SUBSET: s += a2 + " = do_set_pred(c, true, " + a2 + ", " + a + ");"; break;
        case CB_OP_LOOP_INIT:
            s += "{ const Val r_ = " + a + "; if (!qloop_init(c, L" + std::to_string(l) + ", r_, " + std::to_string(I.ib & 0xFF) + ", " + (((I.ib >> 8) & 1) ? "true" : "false") +
                 ", " + std::to_string(I.ia) + ", &" + a + ")) goto " + lab(I.ic - lo) + "; }";
            break;
        case CB_OP_LOOP_NEXT:
            s += "{ const Val r_ = " + a + "; if (!qloop_next(c, L" + std::to_string(l - 1) + ", r_, " + std::to_string(I.ib & 0xFF) + ", " + (((I.ib >> 8) & 1) ? "true" : "false") +
                 ", " + std::to_string(I.ia) + ", &" + a + ")) goto " + lab(I.ic - lo) + "; }";
            break;
        case CB_OP_NOERR: s += a + " = mk_bool(" + a + ".tag != CB_T_ERR);"; break;
        case CB_OP_INT: s += a + " = conv_int(c, " + a + ");"; break;
        case CB_OP_UINT: s += a + " = conv_uint(c, " + a + ");"; break;
        case CB_OP_DOUBLE: s += a + " = op_double(c, " + a + ");"; break;
        case CB_OP_TIMESTAMP: s += a + " = op_timestamp(c, " + a + ");"; break;
        case CB_OP_DURATION: s += a + " = op_duration(c, " + a + ");"; break;
        case CB_OP_DYN: s += ";"; break;
        case CB_OP_CMP_SLOT_CONST: s += top + " = do_cmp(c, " + std::to_string(I.ia) + ", decode_v64(" + slot(I.ib) + ", &st_), " + cst(I.ic) + ");"; break;
        case CB_OP_CMP_SLOT_SLOT: s += "{ const Val x_ = decode_v64(" + slot(I.ib) + ", &st_); " + top + " = do_cmp(c, " + std::to_string(I.ia) + ", x_, decode_v64(" + slot(I.ic) + ", &st_)); }"; break;
        case CB_OP_CMP_SLOT_PID: my_pid = true; s += top + " = do_cmp(c, " + std::to_string(I.ia) + ", decode_v64(" + slot(I.ib) + ", &st_), mk(CB_T_STRING, c.pid));"; break;
        case CB_OP_IN_SLOT_CONST: s += top + " = do_in(c, decode_v64(" + slot(I.ib) + ", &st_), " + cst(I.ic) + ");"; break;
        case CB_OP_IN_CONST_SLOT: s += top + " = do_in(c, " + cst(I.ic) + ", decode_v64(" + slot(I.ib) + ", &st_));"; break;
        case CB_OP_IN_IP_RANGE: s += a + " = " + a + ".tag == CB_T_ERR ? mk_err() : do_in_ip_range(c, " + a + ", c.t->theap() + " + hex(I.ic) + ");"; break;
        case CB_OP_HIER_REL: s += a2 + " = op_hier_rel(c, " + hex(I.ia) + ", " + hex(I.ib) + ", " + hex(I.ic) + ", " + a2 + ", " + a + ");"; break;
        case CB_OP_TS_GET: s += a + " = op_ts_get(c, " + a + ", " + hex(I.ia) + ", " + hex(I.ib) + ", " + hex(I.ic) + ");"; break;
        case CB_OP_IN_SPLIT: s += a2 + " = op_in_split(c, " + a2 + ", " + a + ", " + hex(I.ib) + ");"; break;
        case CB_OP_HIER_SIZE: s += a + " = op_hier_size(c, " + a + ", " + hex(I.ib) + ");"; break;
        case CB_OP_HIER_CA:
            if (I.ia == 0) s += a2 + " = op_hier_ca2(c, " + a2 + ", " + a + ", " + hex(I.ib) + ", " + hex(I.ic) + ");";
            else s += S(d - 3) + " = op_hier_ca3(c, " + S(d - 3) + ", " + a2 + ", " + a + ", " + hex(I.ib) + ", " + hex(I.ic) + ");";
            break;
        case CB_OP_FN: {
            const int base = d - (int)I.ib;
            s += "{ Val a_[" + std::to_string(I.ib) + "] = {";
            for (uint32_t q = 0; q < I.ib; q++) s += std::string(q ? ", " : "") + S(base + (int)q);
            s += "}; " + S(base) + " = op_fn(c, " + hex(I.ia) + ", " + hex(I.ib) + ", a_); }";
            break;
        }
        case CB_OP_MATCHES: s += a + " = op_matches(c, " + a + ", " + hex(I.ic) + ");"; break;
        default: bad = true; break;
        }
        s += "\n";
    }
    if (target[n]) s += lab(n) + ":;\n";
    s += "    return cond_true(s0);\n";
    if (only_slot) *only_slot = my_slots.size() == 1 ? my_slots[0] : CB_NONE32;
    if (reads_pid) *reads_pid = my_pid;
    return bad ? std::string() : s;
}

// A whole condition program -> boolean formula over atoms ("" = does not qualify).  New atoms are appended to `at`.
inline std::string translate_program(const uint32_t *code_words, uint32_t code_off, uint32_t code_len, const uint32_t *consts, uint32_t n_consts, uint32_t n_slots, Atoms &at) {
    if (code_len == 0 || code_len > 4096) return "";
    std::vector<Ins> P(code_len);
    for (uint32_t i = 0; i < code_len; i++) {
        const uint32_t w0 = code_words[2 * (code_off + i)], w1 = code_words[2 * (code_off + i) + 1];
        P[i] = Ins{w0 & 0xFFu, (w0 >> 8) & 0xFFu, w0 >> 16, w1};
    }
    std::vector<std::string> st;    // the condition-level stack, symbolically
    uint32_t i = 0;
    bool ret = false;
    while (i < code_len && !ret) {
        const Ins &I = P[i];
        auto cond_level = [&](uint32_t op) { return op == CB_OP_AND || op == CB_OP_OR || op == CB_OP_COND_NOT || op == CB_OP_RET; };
        switch (I.op) {
        case CB_OP_RET: ret = true; continue;
        case CB_OP_AND: case CB_OP_OR: {
            if (st.size() < 2) return "";
            const std::string b = st.back(); st.pop_back();
            st.back() = "(" + st.back() + (I.op == CB_OP_AND ? " & " : " | ") + b + ")";
            i++;
            continue;
        }
        case CB_OP_COND_NOT: if (st.empty()) return ""; st.back() = "!" + st.back(); i++; continue;
        case CB_OP_JF_KEEP: case CB_OP_JT_KEEP:
            // condition-level short circuit: every leaf is evaluated anyway (no side effects), the formula is what matters
            if (st.empty() || I.ic <= i || I.ic > code_len) return "";
            i++;
            continue;
        default: break;
        }
        // a leaf starts here: it ends at the next TO_COND
        uint32_t e = i;
        while (e < code_len && P[e].op != CB_OP_TO_COND) e++;
        bool literal = false;
        if (I.op == CB_OP_CONST && i + 1 < code_len) {   // all[] / any[] / none[]: a bare constant at condition level
            const uint32_t nx = P[i + 1].op;
            if (cond_level(nx)) literal = true;
            if ((nx == CB_OP_JF_KEEP || nx == CB_OP_JT_KEEP) && (e >= code_len || P[i + 1].ic > e)) literal = true;
        }
        if (literal) {
            if (I.ic >= n_consts || consts[4 * I.ic] != CB_T_BOOL) return "";
            st.push_back(consts[4 * I.ic + 2] ? "true" : "false");
            i++;
            continue;
        }
        if (e >= code_len) return "";
        std::vector<uint32_t> key;
        for (uint32_t k = i; k < e; k++) {
            const Ins &J = P[k];
            const bool j = is_jump(J.op);
            key.push_back(J.op | J.ia << 8 | (J.op == CB_OP_TERN ? (J.ib - i) : J.ib) << 16);
            key.push_back(j ? J.ic - i : J.ic);
        }
        auto it = at.ids.find(key);
        if (it == at.ids.end()) {
            if (at.slot_used.size() < n_slots) at.slot_used.resize(n_slots, false);
            uint32_t one = CB_NONE32;
            bool pid = false;
            const std::string body = atom_source(P, i, e, consts, n_consts, n_slots, at.slot_used, &one, &pid);
            if (body.empty()) return "";
            const uint32_t id = (uint32_t)at.src.size();
            at.only_slot.push_back(one);
            at.reads_pid.push_back(pid);
            at.src.push_back("template <typename Cols>\nCB_HD bool uc_atom_" + std::to_string(id) + "(Ctx &c, const Cols &cols) {\n" + body + "}\n");
            it = at.ids.emplace(key, id).first;
        }
        st.push_back("a" + std::to_string(it->second));
        i = e + 1;
    }
    if (!ret || st.size() != 1) return "";
    return st[0];
}

// ---- unique-condition form (cb_uc.h / cb::eval_request_uc) -----------------------------------------------------------
// For tables whose blocks differ in shape the per-shape inlining above explodes; their DISTINCT conditions are few.
// generate_uc() emits `SpecConds`: load() pulls every attribute slot the conditions read into registers (all loads in
// flight at once, coalesced), operator() evaluates every distinct DNF term once (shared between conditions) and
// combines them into the request's condition word, one bit per condition record of the image (a complement-coded image:
// per base condition, which a condition and its negation share).  Rows stay data (16-byte records walked by cb::uc_walk,
// unrolled over the image's DENY and ALLOW segment slots).
// uc: the compact image (cb_uc.h) and its layout; n_uconds: its distinct conditions (cbuc::Image::n_uconds).  "" = does
// not qualify (a distinct condition without flat form ...).
struct UcLimits {
    uint32_t max_terms = 512;   // distinct terms
};
struct UcSource {
    std::string src;            // "" = does not qualify
    uint32_t n_strpred = 0;     // string predicates served by the per-string pre-pass (BatchView::strpred)
    uint32_t n_atoms = 0;       // leaf programs translated to straight-line code (conditions without a flat form)
};
inline UcSource generate_uc(const uint8_t *uc_image, const uint32_t *off, uint32_t uc_conds_off, uint32_t n_uconds, uint32_t n_slots, uint32_t n_consts = 0,
                            const UcLimits lim = UcLimits()) {
    UcSource out;
    if (n_uconds == 0 || n_uconds > 127) return out;
    const uint32_t *const_words = reinterpret_cast<const uint32_t *>(uc_image + off[CB_SEC_CONSTS]);   // cb_const: {tag, pad, bits}
    Atoms atoms;
    const uint32_t *uconds = reinterpret_cast<const uint32_t *>(uc_image + uc_conds_off);    // [n_bits + 1] x {code_off, code_len, flat_off, flat_info}
    // record 0 (cb_uc.h): {rows the walk visits per scope, DENY slots, ALLOW slots of the segment form (0 / 0: row ranges),
    // complement-coded: the base conditions (one record and one bit each), else 0: one record per distinct condition}
    const uint32_t scope_rows = uconds[0], deny_rows = uconds[1], allow_rows = uconds[2];
    const uint32_t n_bits = uconds[3] ? uconds[3] : n_uconds;
    const uint32_t *base_of = uconds[3] ? uconds + 4 * (n_bits + 1) : nullptr;   // distinct condition - 1 -> base number | negated << 31
    std::vector<std::string> formula(n_bits + 1);   // per condition without flat form: boolean formula over atoms
    const uint32_t *code = reinterpret_cast<const uint32_t *>(uc_image + off[CB_SEC_CODE]);
    const uint64_t *consts = reinterpret_cast<const uint64_t *>(uc_image + off[CB_SEC_CONSTS_V64]);
    const uint64_t *theap = reinterpret_cast<const uint64_t *>(uc_image + off[CB_SEC_THEAP]);
    const uint32_t kUseMask = ~((uint32_t)(CB_TERM_LIT_F | CB_TERM_GROUP_END) << 8);
    std::map<std::vector<uint32_t>, uint32_t> term_ids;
    std::vector<std::vector<uint32_t>> terms;
    const uint32_t ns = n_slots ? n_slots : 1;
    std::vector<bool> slot_used(ns, false), slot_list(ns, false);
    auto is_slot_kind = [](uint32_t kind) { return kind == CB_OPK_SLOT || kind == CB_OPK_SLOT_ELEM || kind == CB_OPK_SLOT_SIZE; };
    auto use_slot = [&](uint32_t kind, uint32_t v) { if (is_slot_kind(kind) && v < ns) slot_used[v] = true; };
    auto v64_tag = [](uint64_t b) { const uint32_t top = (uint32_t)(b >> 48); return (top & 0xFFF0u) == 0xFFF0u ? (top & 0xFu) : 0u; };
    for (uint32_t u = 1; u <= n_bits; u++) {
        const uint32_t *cd = uconds + 4 * u;
        if (cd[3] == 0 || ((cd[3] >> 16) & 0xFF) != CB_FLAT_DNF) {
            formula[u] = translate_program(code, cd[0], cd[1], const_words, n_consts, ns, atoms);
            if (formula[u].empty()) return out;
            continue;
        }
        for (uint32_t i = 0, nt = cd[3] & 0xFFFFu; i < nt; i++) {
            const uint32_t *w = code + 2 * (cd[2] + 2 * i);
            std::vector<uint32_t> key = {w[0] & kUseMask, w[1], w[2], w[3]};
            if (term_ids.emplace(key, (uint32_t)terms.size()).second) terms.push_back(key);
        }
    }
    if (terms.size() > lim.max_terms) return out;
    // per term: which form it takes in the specialised code
    //   'L' list registers (IN with a slot list, set predicates over two slot lists), 'P' string-predicate word, 'G' generic
    std::vector<char> form(terms.size(), 'G');
    std::vector<uint32_t> pred_of(terms.size(), 0);
    std::vector<uint32_t> pred_terms;   // term index of every string predicate
    for (uint32_t q = 0; q < terms.size(); q++) {
        const uint32_t *w = terms[q].data();
        const uint32_t op = w[0] & 0xFF, xk = (w[0] >> 16) & 0xFF, yk = w[0] >> 24;
        switch (op) {   // which operands are slots (bytecode._specialize_term shapes first)
        case CB_TERM_EQ_SS: case CB_TERM_ORD_SS: use_slot(CB_OPK_SLOT, w[1]); use_slot(CB_OPK_SLOT, w[2]); break;
        case CB_TERM_EQ_SC: case CB_TERM_EQ_SP: case CB_TERM_ORD_SC: case CB_TERM_IN_SC: use_slot(CB_OPK_SLOT, w[1]); break;
        case CB_TERM_IN_SS: use_slot(CB_OPK_SLOT, w[1]); use_slot(CB_OPK_SLOT, w[2]); if (w[2] < ns) { slot_list[w[2]] = true; form[q] = 'L'; } break;
        case CB_TERM_IN_CS: use_slot(CB_OPK_SLOT, w[2]); if (w[2] < ns) { slot_list[w[2]] = true; form[q] = 'L'; } break;
        default:
            use_slot(xk, w[1]);
            if (op != CB_TERM_HAS) use_slot(yk, w[2]);
            // size() is read from the list registers: the slot becomes a list slot
            if (xk == CB_OPK_SLOT_SIZE && w[1] < ns) slot_list[w[1]] = true;
            if (op != CB_TERM_HAS && yk == CB_OPK_SLOT_SIZE && w[2] < ns) slot_list[w[2]] = true;
            if (op == CB_TERM_IN && yk == CB_OPK_SLOT && w[2] < ns) { slot_list[w[2]] = true; form[q] = 'L'; }
            if ((op == CB_TERM_INTERSECTS || op == CB_TERM_SUBSET) && xk == CB_OPK_SLOT && yk == CB_OPK_SLOT && w[1] < ns && w[2] < ns) {
                slot_list[w[1]] = slot_list[w[2]] = true;
                form[q] = 'L';
            }
            if ((op == CB_TERM_STARTS || op == CB_TERM_ENDS || op == CB_TERM_CONTAINS) && xk == CB_OPK_SLOT && yk == CB_OPK_CONST &&
                v64_tag(consts[w[2]]) == CB_V64_STRING && pred_terms.size() < 32) {
                form[q] = 'P';
                pred_of[q] = (uint32_t)pred_terms.size();
                pred_terms.push_back(q);
            }
            break;
        }
    }
    // Leaf programs over ONE attribute slot (and nothing else of the request) are functions of that slot's value: for a
    // string value the pre-pass evaluates them once per distinct dictionary string -- timestamp(<claim>) > now(),
    // "x" in <claim>.split(" ") ... -- and the request kernel reads two bits: the value, and "evaluate in place" (the
    // pre-pass met a value the device forms cannot hold: the in-place evaluation then raises it for this request).
    std::vector<int> atom_pred(atoms.src.size(), -1);
    uint32_t n_pred_bits = (uint32_t)pred_terms.size();
    for (uint32_t a = 0; a < atoms.src.size(); a++)
        if (atoms.only_slot[a] != CB_NONE32 && !atoms.reads_pid[a] && n_pred_bits + 2 <= 32) { atom_pred[a] = (int)n_pred_bits; n_pred_bits += 2; }
    // set predicates over two slot lists share one membership mask per list pair (cb_core.h: list_mask): isSubset(A, B)
    // needs "which elements of A occur in B", hasIntersection over the pair takes whichever orientation exists
    std::map<std::pair<uint32_t, uint32_t>, bool> masks;   // (A, B) -> emitted
    std::vector<std::pair<uint32_t, uint32_t>> mask_of(terms.size());
    for (int pass = 0; pass < 2; pass++)
        for (uint32_t q = 0; q < terms.size(); q++) {
            const uint32_t *w = terms[q].data();
            const uint32_t op = w[0] & 0xFF;
            if (form[q] != 'L' || (op != CB_TERM_SUBSET && op != CB_TERM_INTERSECTS) || (op == CB_TERM_SUBSET) != (pass == 0)) continue;
            std::pair<uint32_t, uint32_t> k(w[1], w[2]);
            if (op == CB_TERM_INTERSECTS && !masks.count(k) && masks.count({w[2], w[1]})) k = {w[2], w[1]};
            masks[k] = true;
            mask_of[q] = k;
        }
    auto sl = [](uint32_t v) { return "cols.slot(" + std::to_string(v) + "u)"; };
    // an operand as a value held in registers ("": none -- the generic term path loads it)
    auto operand = [&](uint32_t kind, uint32_t v, uint32_t aux) -> std::string {
        if (kind == CB_OPK_CONST) return hex64(consts[v]);
        if (kind == CB_OPK_PID) return "(((uint64_t)(CB_V64_BOX_BASE | CB_V64_STRING) << 48) | pid)";
        if (v >= ns) return "";
        if (kind == CB_OPK_SLOT) return sl(v);
        const std::string l = "cols.l" + std::to_string(v);
        if (kind == CB_OPK_SLOT_SIZE && slot_list[v]) return "list_size(t, b, " + sl(v) + ", " + l + ")";
        if (kind == CB_OPK_SLOT_ELEM && slot_list[v] && aux < 8) return "list_elem(t, b, " + sl(v) + ", " + l + ", " + std::to_string(aux) + "u)";   // CB_LC
        return "";
    };
    // Membership terms probe their list: each list's distinct scalars (constants, slots, list[i] operands) become keys
    // compared in one pass over the list's elements (cb_core.h: list_probe), right after the loads; the term then reads
    // its hit bit.  At most 32 probes per list (one bit each): further terms probe on their own.
    struct Probe {
        uint32_t kind, v, aux;   // the operand (CB_OPK_*); kind CB_NONE32: one operand() has no register form for
        std::string value;       // its 64-bit value as source text
    };
    auto probe_operand = [&](uint32_t q) -> Probe {
        const uint32_t *w = terms[q].data();
        const uint32_t op = w[0] & 0xFF, xk = (w[0] >> 16) & 0xFF;
        if (op == CB_TERM_IN_CS) return Probe{CB_OPK_CONST, w[1], 0, hex64(consts[w[1]])};
        if (op == CB_TERM_IN_SS) return Probe{CB_OPK_SLOT, w[1], 0, sl(w[1])};
        const std::string x = operand(xk, w[1], w[3] & 0xFFFFu);
        if (!x.empty()) return Probe{xk, w[1], w[3] & 0xFFFFu, x};
        return Probe{CB_NONE32, 0, 0, "uc_term_operand(t, b, cols, pid, " + hex(xk) + ", " + hex(w[1]) + ", " + hex(w[3] & 0xFFFFu) + ")"};
    };
    std::map<uint32_t, std::vector<Probe>> probes;   // list slot -> probe operands
    std::vector<uint32_t> probe_of(terms.size(), CB_NONE32);
    for (uint32_t q = 0; q < terms.size(); q++) {
        const uint32_t op = terms[q][0] & 0xFF;
        if (form[q] != 'L' || (op != CB_TERM_IN_CS && op != CB_TERM_IN_SS && op != CB_TERM_IN)) continue;
        std::vector<Probe> &ps = probes[terms[q][2]];
        const Probe x = probe_operand(q);
        uint32_t p = 0;
        while (p < ps.size() && ps[p].value != x.value) p++;
        if (p == ps.size() && p < 32) ps.push_back(x);
        if (p < ps.size()) probe_of[q] = p;
    }
    auto term_code = [&](uint32_t q) -> std::string {
        const uint32_t *w = terms[q].data();
        const uint32_t op = w[0] & 0xFF, flags = (w[0] >> 8) & 0xFF, xk = (w[0] >> 16) & 0xFF, yk = w[0] >> 24;
        const bool kinds = op <= CB_TERM_SUBSET;   // the generic shapes name their operands' kinds
        const std::string x = kinds ? operand(xk, w[1], w[3] & 0xFFFFu) : "", y = kinds && op != CB_TERM_HAS ? operand(yk, w[2], w[3] >> 16) : "";
        if (form[q] == 'P') return "strpred_tri(b, " + sl(w[1]) + ", " + std::to_string(pred_of[q]) + "u)";
        if (form[q] == 'L') {
            if (op == CB_TERM_IN_CS || op == CB_TERM_IN_SS || op == CB_TERM_IN) {
                const std::string v = std::to_string(w[2]);
                if (probe_of[q] == CB_NONE32) return "list_in_tri(" + probe_operand(q).value + ", cols.l" + v + ", slow)";
                const std::string xp = "x" + v + "_" + std::to_string(probe_of[q]);
                return "list_in_tri(" + xp + ", cols.l" + v + ".st, h" + v + " & " + hex(1u << probe_of[q]) + ", slow)";
            }
            const std::string a = std::to_string(mask_of[q].first), bb = std::to_string(mask_of[q].second);
            return std::string("list_set_tri(") + (op == CB_TERM_SUBSET ? "true" : "false") + ", cols.l" + a + ", cols.l" + bb + ", m" + a + "_" + bb + ", slow)";
        }
        // the shapes term_tri() folds to, and the generic shapes over operands held in registers: the same helpers, called directly
        if (w[1] < ns && w[2] < ns) {
            if (op == CB_TERM_EQ_SS) return "eq_tri(" + sl(w[1]) + ", " + sl(w[2]) + ", slow)";
            if (op == CB_TERM_ORD_SS) return "ord_tri(" + hex(flags & CB_TERM_CI_MASK) + ", " + sl(w[1]) + ", " + sl(w[2]) + ", slow)";
        }
        if (op == CB_TERM_EQ_SP && w[1] < ns) return "eq_tri(" + sl(w[1]) + ", " + operand(CB_OPK_PID, 0, 0) + ", slow)";
        if (op == CB_TERM_HAS && !x.empty()) return "has_tri(" + x + ")";
        if (op == CB_TERM_CMP && !x.empty() && !y.empty()) return "cmp_tri(" + hex(flags & CB_TERM_CI_MASK) + ", " + x + ", " + y + ", slow)";
        if ((op == CB_TERM_STARTS || op == CB_TERM_ENDS || op == CB_TERM_CONTAINS) && !x.empty() && !y.empty())
            return "str_tri(t, b, " + std::to_string(op) + "u, " + x + ", " + y + ")";
        const std::string e = term_expr(w, consts, theap);
        return e.compare(0, 9, "term_tri(") == 0 ? "uc_" + e : e;
    };
    // Slots read by the flat terms live in registers (all loads in flight at once); slots only the leaf programs read --
    // and every slot once the table reads more than kMaxRegSlots of them -- are loaded where they are used (L1-allocating loads).
    const uint32_t kMaxRegSlots = 16;
    const bool have_atoms = !atoms.src.empty();
    atoms.slot_used.resize(ns, false);
    uint32_t n_reg = 0;
    for (uint32_t v = 0; v < ns; v++) n_reg += slot_used[v] || slot_list[v];
    if (n_reg > kMaxRegSlots)
        for (uint32_t v = 0; v < ns; v++) if (!slot_list[v]) slot_used[v] = false;
    // Typed branch: one type per register slot, inferred from the terms that read it -- 'S' string (compared with a
    // string, P.id or another string slot, a string predicate's operand, a probe key), 'N' number (ordered or compared
    // with a number), 'B' bool (compared with a bool), 'L' cached list.  When every register slot has exactly one type,
    // load() keeps the slots as typed payloads plus a per-request guard (cb_core.h: typed_*), and every term becomes a
    // plain boolean under that guard; lanes that fail it evaluate today's tri-state terms on their reloaded slot words.
    std::vector<char> ty(ns, 0);
    std::vector<uint32_t> list_need(ns, 0);   // per list slot: 1 + the largest constant index read from it
    bool typed = n_reg > 0 && n_reg <= kMaxRegSlots;
    auto want = [&](uint32_t v, char k) {   // k = 0: an operand no typed term can take
        if (v >= ns || !k) { typed = false; return; }
        if (ty[v] && ty[v] != k) typed = false;
        ty[v] = k;
    };
    auto const_type = [&](uint64_t c) -> char {
        const uint32_t tag = v64_tag(c);
        double d;
        memcpy(&d, &c, sizeof d);
        if (tag == 0) return d == d ? 'N' : 0;   // a NaN constant orders as an error
        if (tag == CB_V64_STRING) return (uint32_t)(c >> 32) == (uint32_t)(CB_V64_BOX_BASE | CB_V64_STRING) << 16 ? 'S' : 0;
        if (tag == CB_V64_BOOL) return (c >> 1) == (uint64_t)(CB_V64_BOX_BASE | CB_V64_BOOL) << 47 ? 'B' : 0;
        return 0;
    };
    // the type an operand of a generic shape names (0: none a typed term can take); slots get it through want()
    auto operand_type = [&](uint32_t kind, uint32_t v, uint32_t aux) -> char {
        if (kind == CB_OPK_CONST) return const_type(consts[v]);
        if (kind == CB_OPK_PID) return 'S';
        if (v >= ns || !slot_list[v] || (kind == CB_OPK_SLOT_ELEM && aux >= 8)) return kind == CB_OPK_SLOT ? 0 : 'X';
        if (kind == CB_OPK_SLOT_SIZE) return 'N';
        if (kind == CB_OPK_SLOT_ELEM) { list_need[v] = aux + 1 > list_need[v] ? aux + 1 : list_need[v]; return 'S'; }
        return 0;
    };
    // x in [constants]: the elements' one type (0: mixed, a NaN or a container, or more than term_expr() inlines)
    auto in_const_type = [&](uint32_t q) -> char {
        const uint64_t *p = theap + (consts[terms[q][2]] & 0xFFFFFFFFFFFFull);
        if (p[0] == 0 || p[0] > 16) return 0;
        char k = const_type(p[1]);
        for (uint32_t j = 1; j < (uint32_t)p[0]; j++) k = const_type(p[1 + j]) == k ? k : 0;
        return k == 'S' || k == 'N' ? k : 0;
    };
    for (uint32_t q = 0; q < terms.size() && typed; q++) {
        const uint32_t *w = terms[q].data();
        const uint32_t op = w[0] & 0xFF, xk = (w[0] >> 16) & 0xFF, yk = w[0] >> 24;
        switch (op) {
        case CB_TERM_EQ_SS: case CB_TERM_ORD_SS: break;   // typed by their other terms
        case CB_TERM_EQ_SC: want(w[1], const_type(consts[w[2]])); break;
        case CB_TERM_ORD_SC: want(w[1], const_type(consts[w[2]]) == 'N' ? 'N' : 0); break;
        case CB_TERM_EQ_SP: want(w[1], 'S'); break;
        case CB_TERM_IN_SC: want(w[1], in_const_type(q)); break;
        case CB_TERM_IN_SS: want(w[1], 'S'); want(w[2], 'L'); break;
        case CB_TERM_IN_CS: want(w[2], 'L'); break;
        default: {
            if (op == CB_TERM_HAS) { if (xk != CB_OPK_SLOT) typed = false; break; }
            const char tx = operand_type(xk, w[1], w[3] & 0xFFFFu), tyy = operand_type(yk, w[2], w[3] >> 16);
            if (tx == 'X' || tyy == 'X') { typed = false; break; }
            if (form[q] == 'L') {
                if (op == CB_TERM_IN) { if (xk == CB_OPK_SLOT) want(w[1], 'S'); want(w[2], 'L'); }
                else { want(w[1], 'L'); want(w[2], 'L'); }
                break;
            }
            if (op == CB_TERM_STARTS || op == CB_TERM_ENDS || op == CB_TERM_CONTAINS) {
                if (xk == CB_OPK_SLOT) want(w[1], 'S');
                if (yk == CB_OPK_SLOT) want(w[2], 'S');
                break;
            }
            // CMP: a slot takes the type of what it is compared with
            if (xk == CB_OPK_SLOT && yk != CB_OPK_SLOT) want(w[1], tyy);
            if (yk == CB_OPK_SLOT && xk != CB_OPK_SLOT) want(w[2], tx);
            break;
        }
        }
    }
    for (uint32_t v = 0; v < ns && typed; v++) {
        if (slot_list[v]) want(v, 'L');
        if ((slot_used[v] || slot_list[v]) && (!ty[v] || atoms.slot_used[v])) typed = false;   // untyped, or leaf programs read the word
    }
    // a scalar operand as source text of its payload type: string id 'S', double 'N', bool 'B' (k = 0, "": not a scalar
    // the typed branch holds -- a list slot, a constant of another type)
    auto typed_operand = [&](uint32_t kind, uint32_t v, uint32_t aux, char &k) -> std::string {
        const std::string V = std::to_string(v);
        if (kind == CB_OPK_CONST) {
            const uint64_t c = consts[v];
            k = const_type(c);
            if (k == 'S') return hex((uint32_t)c);
            if (k == 'N') return "u2d(" + hex64(c) + ")";
            if (k == 'B') return c & 1u ? "true" : "false";
            return "";
        }
        if (kind == CB_OPK_PID) { k = 'S'; return "pid"; }
        if (kind == CB_OPK_SLOT_SIZE) { k = 'N'; return "(double)cols.l" + V + ".len"; }
        if (kind == CB_OPK_SLOT_ELEM) { k = 'S'; return "typed_id(cols.l" + V + ".e[" + std::to_string(aux) + "])"; }
        k = v < ns && (ty[v] == 'S' || ty[v] == 'N' || ty[v] == 'B') ? ty[v] : 0;
        return k == 'S' ? "typed_id(cols.k" + V + ")" : k == 'N' ? "cols.d" + V : k == 'B' ? "cols.b" + V : "";
    };
    // per term: the plain boolean it is under the guard ("" = no typed form: the table gets no typed branch)
    auto typed_term = [&](uint32_t q) -> std::string {
        const uint32_t *w = terms[q].data();
        const uint32_t op = w[0] & 0xFF, flags = (w[0] >> 8) & 0xFF, xk = (w[0] >> 16) & 0xFF, yk = w[0] >> 24, ci = flags & CB_TERM_CI_MASK;
        if (form[q] == 'P') return "typed_strpred(b, typed_id(cols.k" + std::to_string(w[1]) + "), " + std::to_string(pred_of[q]) + "u)";
        if (form[q] == 'L') {
            if (op == CB_TERM_IN_CS || op == CB_TERM_IN_SS || op == CB_TERM_IN) {
                if (probe_of[q] == CB_NONE32) return "";
                if (op == CB_TERM_IN_CS && const_type(consts[w[1]]) == 0) return "";   // NaN / null / containers: not a plain membership
                if (op == CB_TERM_IN && xk == CB_OPK_CONST && const_type(consts[w[1]]) == 0) return "";
                return "(h" + std::to_string(w[2]) + " & " + hex(1u << probe_of[q]) + ") != 0u";
            }
            const std::string a = std::to_string(mask_of[q].first), bb = std::to_string(mask_of[q].second);
            return op == CB_TERM_SUBSET ? "m" + a + "_" + bb + " == (1u << cols.l" + a + ".len) - 1u" : "m" + a + "_" + bb + " != 0u";
        }
        char kx = 0, ky = 0;
        std::string x, y;
        switch (op) {
        case CB_TERM_EQ_SS: case CB_TERM_ORD_SS:
            x = typed_operand(CB_OPK_SLOT, w[1], 0, kx); y = typed_operand(CB_OPK_SLOT, w[2], 0, ky);
            if (!kx || kx != ky) return "";   // list == list: containers, the tri-state terms defer them
            if (op == CB_TERM_EQ_SS) return x + " == " + y;
            return kx == 'N' ? "typed_ord(" + hex(ci) + ", " + x + ", " + y + ")" : "";
        case CB_TERM_EQ_SC: case CB_TERM_ORD_SC:
            x = typed_operand(CB_OPK_SLOT, w[1], 0, kx); y = typed_operand(CB_OPK_CONST, w[2], 0, ky);
            if (!kx || kx != ky) return "";
            if (op == CB_TERM_EQ_SC) return x + " == " + y;
            return kx == 'N' ? "typed_ord(" + hex(ci) + ", " + x + ", " + y + ")" : "";
        case CB_TERM_EQ_SP: return "typed_id(cols.k" + std::to_string(w[1]) + ") == pid";
        case CB_TERM_IN_SC: {
            const uint64_t *p = theap + (consts[w[2]] & 0xFFFFFFFFFFFFull);
            x = typed_operand(CB_OPK_SLOT, w[1], 0, kx);
            if (!kx || kx != in_const_type(q)) return "";
            std::string e;
            for (uint32_t j = 0; j < (uint32_t)p[0]; j++)
                e += std::string(j ? " | " : "") + "(" + x + " == " + (kx == 'S' ? hex((uint32_t)p[1 + j]) : "u2d(" + hex64(p[1 + j]) + ")") + ")";
            return e;
        }
        case CB_TERM_HAS: return "true";
        case CB_TERM_CMP:
            x = typed_operand(xk, w[1], w[3] & 0xFFFFu, kx); y = typed_operand(yk, w[2], w[3] >> 16, ky);
            if (!kx || !ky) return "";
            if (ci == 0) return kx == ky ? x + " == " + y : "false";   // scalars of two types are not equal
            return kx == 'N' && ky == 'N' ? "typed_ord(" + hex(ci) + ", " + x + ", " + y + ")" : "";
        case CB_TERM_STARTS: case CB_TERM_ENDS: case CB_TERM_CONTAINS:
            x = typed_operand(xk, w[1], w[3] & 0xFFFFu, kx); y = typed_operand(yk, w[2], w[3] >> 16, ky);
            if (kx != 'S' || ky != 'S') return "";
            return "str_tri(t, b, " + std::to_string(op) + "u, typed_box(" + x + "), typed_box(" + y + ")) == TRI_T";
        default: return "";
        }
    };
    std::vector<std::string> tterm(terms.size());
    for (uint32_t q = 0; q < terms.size() && typed; q++) {
        tterm[q] = typed_term(q);
        typed = !tterm[q].empty();
    }
    // probe keys from the typed registers ("": none): a string slot's register is its probe key, an element of a list
    // its key without the slot word (cb_core.h: list_elem_key), a constant's or P.id's key folds
    auto probe_key = [&](const Probe &x) -> std::string {
        const std::string V = std::to_string(x.v);
        if (x.kind == CB_OPK_CONST || x.kind == CB_OPK_PID) return "list_probe_key(" + x.value + ")";
        if (x.kind == CB_OPK_SLOT) return x.v < ns && ty[x.v] == 'S' ? "cols.k" + V : "";
        if (x.kind == CB_OPK_SLOT_ELEM) return "list_elem_key(t, b, cols, " + V + "u, cols.l" + V + ", " + std::to_string(x.aux) + "u)";
        return "";
    };
    for (const auto &pl : probes)
        for (const Probe &x : pl.second) typed &= !probe_key(x).empty();
    std::string s;
    s += "// generated by cb_specialize.h (generate_uc) from the loaded table: every distinct condition, straight-line\n";
    s += "namespace cb {\n";
    for (const std::string &a : atoms.src) s += a;
    auto reg = [&](uint32_t v) { return slot_used[v] || slot_list[v]; };
    s += "struct SpecRegs {\n    CachedCols g;\n";
    for (uint32_t v = 0; v < ns; v++)
        if (reg(v)) s += "    uint64_t s" + std::to_string(v) + ";\n";
    if (typed) {
        // the words above are read by load() alone (slot() reloads them): only the typed payloads live on
        s += "    bool typed;   // every slot below holds the type its terms compare it as (SpecConds::load)\n";
        for (uint32_t v = 0; v < ns; v++) {
            const std::string V = std::to_string(v);
            if (ty[v] == 'S') s += "    ListKey k" + V + ";   // string: its probe key (the id when typed)\n";
            if (ty[v] == 'N') s += "    double d" + V + ";\n";
            if (ty[v] == 'B') s += "    bool b" + V + ";\n";
        }
    }
    for (uint32_t v = 0; v < ns; v++)
        if (slot_list[v]) s += "    ListRegs l" + std::to_string(v) + ";\n";
    s += "    CB_HD uint64_t slot(uint32_t v) const {\n        switch (v) {\n";
    for (uint32_t v = 0; v < ns && !typed; v++)
        if (reg(v)) s += "        case " + std::to_string(v) + "u: return s" + std::to_string(v) + ";\n";
    s += "        default: return v < " + std::to_string(ns) + "u ? g.slot(v) : (uint64_t)(CB_V64_BOX_BASE | CB_V64_ERROR) << 48;\n        }\n    }\n};\n";
    s += "struct SpecConds {\n    static constexpr uint32_t n_strpred = " + std::to_string(n_pred_bits) + "u;\n";
    s += std::string("    static constexpr int kForm = ") + (n_bits <= 31 ? "CB_UC_FORM_MASK32" : n_bits <= 63 ? "CB_UC_FORM_MASK64" : "CB_UC_FORM_INDEX") + ";   // how the rows name their conditions\n";
    if (base_of) {   // complement-coded image: the rows need each base condition true or false
        s += "    // " + std::to_string(n_uconds) + " distinct conditions on " + std::to_string(n_bits) + " base conditions, one bit each:\n";
        for (uint32_t d = 0; d < n_uconds; d++)
            s += "    // distinct condition " + std::to_string(d + 1) + ": " + (base_of[d] >> 31 ? "!" : "") + "base condition " + std::to_string(base_of[d] & 0x7FFFFFFFu) + "\n";
    }
    s += "    static constexpr uint32_t kScopeRows = " + std::to_string(scope_rows) + "u;   // rows the walk visits per scope (cb::uc_walk)\n";
    s += "    static constexpr uint32_t kDenyRows = " + std::to_string(deny_rows) + "u, kAllowRows = " + std::to_string(allow_rows) +
         "u;   // segment slots (0 / 0: row ranges)\n";
    s += std::string("    static constexpr bool kPrograms = ") + (have_atoms ? "true" : "false") + ";   // leaf programs: needs the value helpers of cb_core.h\n";
    {   // the slots load() keeps as register-resident lists: the kernel prefetches their headers a chunk ahead.  Not for
        // tables with leaf programs (2 CTAs / SM and a stack frame): on C5 the prefetch made the kernel slower (DESIGN §7)
        std::string ls;
        uint32_t nls = 0;
        for (uint32_t v = 0; v < ns && !have_atoms; v++)
            if (slot_list[v]) ls += (nls++ ? ", " : "") + std::to_string(v) + "u";
        s += "    static constexpr uint32_t kListSlots = " + std::to_string(nls) + "u;   // list slots whose headers check_uc_body prefetches\n";
        s += "    static constexpr uint32_t kListSlot[" + std::to_string(nls ? nls : 1u) + "] = {" + (nls ? ls : "0u") + "};\n";
    }
    s += "    template <typename Cols>\n    CB_HD SpecRegs load(const TableView t, const BatchView &b, const Cols &c) const {\n        SpecRegs r;\n        r.g.b = c.b; r.g.n = c.n;\n";
    for (uint32_t v = 0; v < ns; v++)
        if (reg(v)) s += "        r.s" + std::to_string(v) + " = c.slot(" + std::to_string(v) + "u);\n";
    if (typed) {
        // the slot words die here: what stays live is the typed payloads and the guard
        std::string guard;
        for (uint32_t v = 0; v < ns; v++) {
            const std::string V = std::to_string(v);
            if (!reg(v)) continue;
            if (ty[v] == 'L') s += "        r.l" + V + " = list_load(t, b, r.s" + V + ");\n";
            if (ty[v] == 'S') s += "        r.k" + V + " = list_probe_key(r.s" + V + ");\n";
            if (ty[v] == 'N') s += "        r.d" + V + " = u2d(r.s" + V + ");\n";
            if (ty[v] == 'B') s += "        r.b" + V + " = (r.s" + V + " & 1u) != 0;\n";
            guard += std::string(guard.empty() ? "" : " & ") + (ty[v] == 'L' ? "typed_list(r.l" + V + ", " + std::to_string(list_need[v]) + "u)"
                                                                 : std::string(ty[v] == 'S' ? "typed_str" : ty[v] == 'N' ? "typed_num" : "typed_bool") + "(r.s" + V + ")");
        }
        s += "        r.typed = " + guard + ";\n";
    } else {
        for (uint32_t v = 0; v < ns; v++)
            if (slot_list[v]) s += "        r.l" + std::to_string(v) + " = list_load(t, b, r.s" + std::to_string(v) + ");\n";
    }
    s += "        return r;\n    }\n";
    s += "    // the predicate word of one string (pre-pass over the string dictionary; bit p = predicate p holds)\n";
    s += "    CB_HD uint32_t strpred(const TableView t, const BatchView &b, uint32_t id) const {\n";
    s += "        OneCols cols; cols.x = ((uint64_t)(CB_V64_BOX_BASE | CB_V64_STRING) << 48) | id;\n        bool slow = false; uint32_t bits = 0u; const uint32_t pid = 0u;\n";
    for (uint32_t p = 0; p < pred_terms.size(); p++) {
        const uint32_t *w = terms[pred_terms[p]].data();
        s += "        bits |= (uint32_t)(term_tri(t, b, cols, pid, U4{" + hex(w[0]) + ", 0x0u, " + hex(w[2]) + ", " + hex(w[3]) + "}, slow) == TRI_T) << " + std::to_string(p) + ";\n";
    }
    {
        bool any = false;
        for (int p : atom_pred) any |= p >= 0;
        if (any) {
            s += "        Ctx c; c.t = &t; c.b = &b; c.req = 0; c.pid = 0; c.edr = 0;\n";
            for (uint32_t a = 0; a < atoms.src.size(); a++)
                if (atom_pred[a] >= 0)
                    s += "        c.unsupported = 0; c.scr_used = 0; bits |= (uint32_t)uc_atom_" + std::to_string(a) + "(c, cols) << " + std::to_string(atom_pred[a]) +
                         "; bits |= (uint32_t)(c.unsupported != 0) << " + std::to_string(atom_pred[a] + 1) + ";\n";
        }
    }
    s += "        (void)slow; (void)pid;\n        return bits;\n    }\n";
    s += "    CB_HD CondWord operator()(const TableView t, const BatchView &b, const SpecRegs &cols, uint32_t pid, uint64_t n, bool &slow) const {\n";
    // the list terms first: after them only the lists' st / len and the elements that list[i] operands read stay live
    // (typed: the keys come from the registers, the probe operands' values only in the tri-state branch)
    const std::string in = typed ? "            " : "        ";
    for (const auto &pl : probes) {
        const std::string v = std::to_string(pl.first);
        std::string keys;
        for (uint32_t p = 0; p < pl.second.size(); p++) {
            const std::string xp = "x" + v + "_" + std::to_string(p);
            if (!typed) s += "        const uint64_t " + xp + " = " + pl.second[p].value + ";\n";
            keys += std::string(p ? ", " : "") + (typed ? probe_key(pl.second[p]) : "list_probe_key(" + xp + ")");
        }
        s += "        const ListKey k" + v + "[" + std::to_string(pl.second.size()) + "] = {" + keys + "};\n";
        s += "        const uint32_t h" + v + " = list_probe(cols.l" + v + ", k" + v + ");   // bit p: x" + v + "_p is an element of slot " + v + "\n";
    }
    for (const auto &m : masks) {
        const std::string a = std::to_string(m.first.first), bb = std::to_string(m.first.second);
        s += "        const uint32_t m" + a + "_" + bb + " = list_mask(cols.l" + a + ", cols.l" + bb + ");   // elements of slot " + a + " in slot " + bb + "\n";
    }
    std::string tri;   // the tri-state terms and conditions (the whole evaluator without the typed branch)
    if (typed)
        for (const auto &pl : probes)
            for (uint32_t p = 0; p < pl.second.size(); p++)
                tri += in + "const uint64_t x" + std::to_string(pl.first) + "_" + std::to_string(p) + " = " + pl.second[p].value + ";\n";
    for (int list_terms = 1; list_terms >= 0; list_terms--)
        for (uint32_t q = 0; q < terms.size(); q++)
            if ((form[q] == 'L') == (list_terms == 1)) tri += in + "const int q" + std::to_string(q) + " = " + term_code(q) + ";\n";
    std::string atom_src;
    if (have_atoms) {
        atom_src += "        Ctx c; c.t = &t; c.b = &b; c.req = n; c.pid = pid; c.unsupported = 0; c.edr = 0; c.scr_used = 0;\n";
        for (uint32_t a = 0; a < atoms.src.size(); a++) {
            const std::string A = std::to_string(a);
            if (atom_pred[a] >= 0) {
                const std::string P = std::to_string(atom_pred[a]), V = sl(atoms.only_slot[a]);
                atom_src += "        bool a" + A + ";\n        {\n            const uint64_t x = " + V + ";\n            const uint32_t w = v64_tag(x) == CB_V64_STRING && !v64_bad(x) ? ldg(b.strpred + (uint32_t)(x & 0xFFFFFFFFu)) >> " + P + " : 2u;\n";
                atom_src += "            if (w & 2u) { c.scr_used = 0; a" + A + " = uc_atom_" + A + "(c, cols); } else a" + A + " = (w & 1u) != 0;\n        }\n";
            } else {
                atom_src += "        c.scr_used = 0; const bool a" + A + " = uc_atom_" + A + "(c, cols);\n";
            }
        }
        atom_src += "        slow |= c.unsupported != 0;   // a value the device forms cannot hold: the general kernel reports it\n";
    } else atom_src += "        (void)n;\n";
    std::string typed_src;
    std::vector<std::string> cond_src(n_bits + 1);   // per condition bit: its tri-state block, or its program line
    // the bit of each record; in the 32-bit form the upper half of the word stays zero
    const std::string what = base_of ? "base condition " : "distinct condition ", cast = n_bits <= 31 ? "(uint32_t)" : "(uint64_t)";
    if (typed) {
        typed_src += "        if (uc_typed(cols.typed)) {   // every term a plain boolean: no error, no deferral\n";
        for (uint32_t q = 0; q < terms.size(); q++) typed_src += "            const bool t" + std::to_string(q) + " = " + tterm[q] + ";\n";
    }
    for (uint32_t u = 1; u <= n_bits; u++) {
        const uint32_t *cd = uconds + 4 * u;
        const std::string word = u < 64 ? "val.lo" : "val.hi", sh = std::to_string(u & 63u);
        if (!formula[u].empty()) {
            cond_src[u] = "        " + word + " |= " + cast + "(" + formula[u] + ") << " + sh + ";   // " + what + std::to_string(u) + " (program)\n";
            continue;
        }
        const uint32_t nt = cd[3] & 0xFFFFu, negate = (cd[3] >> 24) & 1u;
        std::string &c = cond_src[u];
        c += in + "{   // " + what + std::to_string(u) + "\n" + in + "    bool any = false, group = true;\n";
        std::string any, group;   // typed: an OR of ANDs of literals
        for (uint32_t i = 0; i < nt; i++) {
            const uint32_t *w = code + 2 * (cd[2] + 2 * i);
            const uint32_t flags = (w[0] >> 8) & 0xFFu;
            const uint32_t q = term_ids[{w[0] & kUseMask, w[1], w[2], w[3]}];
            c += in + "    group &= term_lit(q" + std::to_string(q) + ", " + hex(flags) + ");\n";
            group += std::string(group.empty() ? "" : " & ") + (flags & CB_TERM_LIT_F ? "!t" : "t") + std::to_string(q);
            if (flags & CB_TERM_GROUP_END) {
                c += in + "    any |= group; group = true;\n";
                any += std::string(any.empty() ? "" : " | ") + "(" + group + ")";
                group.clear();
            }
        }
        c += in + "    " + word + " |= " + cast + "(any != " + (negate ? "true" : "false") + ") << " + sh + ";\n" + in + "}\n";
        if (any.empty()) any = "false";
        typed_src += "            " + word + " |= " + cast + "(" + (negate ? "!(" + any + ")" : any) + ") << " + sh + ";   // " + (base_of ? what : std::string("condition ")) + std::to_string(u) + "\n";
    }
    if (typed) {
        s += atom_src + "        CondWord val; val.lo = 1ull; val.hi = 0ull;\n" + typed_src + "        } else {   // the tri-state terms on the slot words, reloaded (cols.slot)\n" + tri;
        for (uint32_t u = 1; u <= n_bits; u++) if (formula[u].empty()) s += cond_src[u];
        s += "        }\n";
        for (uint32_t u = 1; u <= n_bits; u++) if (!formula[u].empty()) s += cond_src[u];
    } else {
        s += tri + atom_src + "        CondWord val; val.lo = 1ull; val.hi = 0ull;\n";
        for (uint32_t u = 1; u <= n_bits; u++) s += cond_src[u];
    }
    s += "        return val;\n    }\n};\n}  // namespace cb\n";
    out.src = s;
    out.n_strpred = n_pred_bits;
    out.n_atoms = (uint32_t)atoms.src.size();
    return out;
}

}  // namespace cbspec
