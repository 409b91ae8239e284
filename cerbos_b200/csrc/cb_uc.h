// cb_uc.h -- host-side builder of the "unique condition" image of a loaded table.
//
// The flattened table (cerbos_b200/table/flatten.py) keeps one condition list per policy block, the way the reference
// keeps one compiled condition per rule (ruletable.go:105-416).  Across a policy set the same conditions recur: shared
// derived roles, the same ownership / tenancy test on every resource kind.  This builder
//   * numbers the DISTINCT conditions of the table 1..U (same DNF term list, or -- no flat form -- same bytecode program),
//     or, where that fits 31 bits, their BASE conditions (a condition and its negation share one, see build()),
//   * rewrites every row to {original index, role, effect, masks of the condition bits it needs} (16 bytes, DENY rows first
//     per block) and, where they fit, lays the rows out in fixed per-block DENY and ALLOW segments of slots,
//   * copies only the sections the unique-condition kernels read into a compact image (C3: 49 KB blob -> ~10 KB),
// so that a kernel can evaluate every distinct condition of a request once, with all lanes in lock step, and walk the
// rows as mask algebra (cb::eval_request_uc).  Built once per cgpu_table_load; the Python blob format is unchanged.
//
// Host-only, no CUDA dependencies: tests/hostsim uses it too.
#pragma once
#include <stdint.h>

#include <cstring>
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "cb_core.h"

namespace cbuc {

constexpr uint32_t kMaxUconds = 127;      // bit 0 of the condition word is "no condition"
constexpr uint32_t kMaxMaskUconds = 63;   // up to here rows carry need MASKS; above, the two condition NUMBERS (cb_core.h: CB_UC_FORM_INDEX)
constexpr uint32_t kMaxComplementBits = 31;   // complement-coded rows: base conditions of one 32-bit condition word
constexpr uint32_t kNegated = 1u << 31;   // ucond_of_gid: the condition holds where its base condition does not

struct Image {
    bool ok = false;
    std::string why;                    // when !ok
    std::vector<uint8_t> bytes;         // compact image (16-byte aligned sections)
    cb::TableLayout lay{};              // offsets into `bytes` + the dims of the source layout
    uint32_t n_uconds = 0, n_flat = 0;  // distinct conditions; how many of them have a flat (DNF) form
    uint32_t n_bits = 0;                // condition records of the image, one bit of the condition word each (see build())
    bool complement = false;            // the records are base conditions: rows need each of theirs true or false
    // programs among the conditions, or rows in index form: only the run-time specialised kernel can evaluate the image
    bool needs_spec() const { return n_flat != n_uconds || n_bits > kMaxMaskUconds; }
    uint32_t scope_rows = 0;            // rows the walk visits in one scope: deny_rows + allow_rows, else the longest row range
    uint32_t deny_rows = 0, allow_rows = 0;   // slots of every block's DENY / ALLOW segment (0 / 0: row ranges, see build())
    uint32_t n_gids = 0, n_gids_flat = 0;   // table conditions (per-block lists), and how many of them have a flat form
    std::vector<uint32_t> ucond_of_gid; // table condition id -> its condition bit (1..n_bits), | kNegated: it needs the bit clear
};

// image: the table image (blob bytes); off / len: section offset and byte length by section id; lay: its layout
inline Image build(const uint8_t *image, const uint32_t *off, const uint64_t *len, const uint32_t *meta, const cb::TableLayout &lay) {
    Image out;
    const uint32_t n_blocks = meta[CB_META_N_BLOCKS], n_rows = meta[CB_META_N_ROWS], n_conds = meta[CB_META_N_CONDS];
    if (n_blocks == 0) { out.why = "no policy blocks"; return out; }
    if (lay.nR > 64) { out.why = "more than 64 roles"; return out; }
    const uint32_t *blocks = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_BLOCKS]);
    const uint32_t *rows = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_ROWS]);
    const uint32_t *conds = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_CONDS]);
    if (len[CB_SEC_BLOCKS] < (uint64_t)n_blocks * 16 || len[CB_SEC_ROWS] < (uint64_t)n_rows * 16 || len[CB_SEC_CONDS] < (uint64_t)n_conds * 16) {
        out.why = "section sizes do not match META";
        return out;
    }
    // Distinct conditions: the same DNF term list (flat_off, flat_info), or -- no flat form -- the same bytecode program.
    // A flat condition and its final negation (flat_info's negate bit: a top-level `none`, as the REQUIRE_PARENTAL_CONSENT
    // scopes wrap their conditional ALLOWs) share one BASE condition.  The negation is exact, errors included: a term that
    // fails is neither true nor false as a literal, so the DNF's `any` is false and `none` holds, as in the reference
    // (ruletable.go:1425-1441: a failed evaluation does not satisfy; none = not any).  When the base conditions fit one
    // 32-bit word (bit 0: "no condition") and some condition is negated, the image is COMPLEMENT-coded: one record and one
    // bit per base condition, and a row needs each of its conditions true (first mask) or false (second mask).  Otherwise
    // one record and one bit per distinct condition, negated or not, as rows of up to 63 bits of masks or in index form.
    std::map<std::tuple<uint32_t, uint32_t, uint32_t>, uint32_t> ids, base_ids;
    std::vector<uint32_t> rec_distinct, rec_base;   // 4 words per distinct / base condition: {code_off, code_len, flat_off, flat_info}
    std::vector<uint32_t> ucond_of, base_of;        // table condition id -> distinct number; distinct number - 1 -> base number | kNegated
    ucond_of.assign(n_conds, 0);
    for (uint32_t g = 0; g < n_conds; g++) {
        const uint32_t *cd = conds + 4 * g;   // {code_off, code_len, flat_off, flat_info}
        const bool flat = cd[3] != 0 && ((cd[3] >> 16) & 0xFF) == CB_FLAT_DNF;
        const auto key = flat ? std::make_tuple(1u, cd[2], cd[3]) : std::make_tuple(0u, cd[0], cd[1]);
        auto it = ids.find(key);
        if (it == ids.end()) {
            const uint32_t u = (uint32_t)ids.size() + 1;
            if (u > kMaxUconds) { out.why = "more than 127 distinct conditions"; return out; }
            it = ids.emplace(key, u).first;
            rec_distinct.insert(rec_distinct.end(), {cd[0], cd[1], flat ? cd[2] : 0u, flat ? cd[3] : 0u});
            out.n_flat += flat;
            const uint32_t neg = flat ? cd[3] & 1u << 24 : 0u;
            const auto bkey = flat ? std::make_tuple(1u, cd[2], cd[3] & ~neg) : key;
            auto bt = base_ids.find(bkey);
            if (bt == base_ids.end()) {
                bt = base_ids.emplace(bkey, (uint32_t)base_ids.size() + 1).first;
                rec_base.insert(rec_base.end(), {cd[0], cd[1], flat ? cd[2] : 0u, flat ? cd[3] & ~neg : 0u});
            }
            base_of.push_back(bt->second | (neg ? kNegated : 0u));
        }
        ucond_of[g] = it->second;
        out.n_gids++;
        out.n_gids_flat += flat;
    }
    out.n_uconds = (uint32_t)ids.size();
    out.complement = base_ids.size() < ids.size() && base_ids.size() <= kMaxComplementBits;
    out.n_bits = out.complement ? (uint32_t)base_ids.size() : out.n_uconds;
    out.ucond_of_gid.assign(n_conds, 0);
    for (uint32_t g = 0; g < n_conds; g++) out.ucond_of_gid[g] = out.complement ? base_of[ucond_of[g] - 1] : ucond_of[g];
    // the condition section: entry 0 {scope_rows, deny_rows, allow_rows, complement-coded: n_bits, else 0}, one record per
    // bit, then (complement-coded) one word per distinct condition, base number | kNegated, for the generator's listing
    std::vector<uint32_t> ucond_rec(4, 0);
    const std::vector<uint32_t> &recs = out.complement ? rec_base : rec_distinct;
    ucond_rec.insert(ucond_rec.end(), recs.begin(), recs.end());
    if (out.complement) ucond_rec.insert(ucond_rec.end(), base_of.begin(), base_of.end());
    // Conditions without a flat form stay in the image as programs: only the run-time specialised kernel evaluates them
    // (cb_specialize.h turns their bytecode into straight-line code); the generic unique-condition kernels defer such
    // requests, so the library uses the image of a table with programs only once its specialised kernel is loaded.
    // rows: DENY rows first inside every block (within a scope every matching row is evaluated and DENY beats ALLOW,
    // ruletable.go:1083-1118, so the order of rows inside a block is free); 16 bytes each, see cb_core.h.  Words 2 / 3:
    // the 64-bit need mask (bit 0 always set), or complement-coded the need-true mask (bit 0 always set) and the
    // need-false mask, or in index form the two condition numbers
    std::vector<uint32_t> urows(4 * (size_t)(n_rows ? n_rows : 1), 0);
    std::vector<uint32_t> ublocks(blocks, blocks + 4 * (size_t)n_blocks);   // {row_start, n_rows, DENY rows, 0}
    const bool index_form = out.n_bits > kMaxMaskUconds;
    for (uint32_t b = 0; b < n_blocks; b++) {
        const uint32_t *bl = blocks + 4 * b;   // {row_start, n_rows, cond_base, n_conds}
        if ((uint64_t)bl[0] + bl[1] > n_rows || (uint64_t)bl[2] + bl[3] > n_conds) { out.why = "block out of range"; return out; }
        uint32_t at = bl[0], n_deny = 0;
        for (int pass = 0; pass < 2; pass++) {
            for (uint32_t r = 0; r < bl[1]; r++) {
                const uint32_t *row = rows + 4 * (bl[0] + r);
                const uint32_t role = row[0] & 0xFFFFu, c = row[0] >> 16, dc = row[1] & 0xFFFFu, effect = row[2] & 0xFFu;
                if ((effect == CB_EFFECT_DENY) != (pass == 0)) continue;
                if ((c && c > bl[3]) || (dc && dc > bl[3])) { out.why = "row condition out of range"; return out; }
                if (role != CB_ROLE_ANY && role >= 64) { out.why = "role id out of range"; return out; }
                const uint32_t uc = c ? out.ucond_of_gid[bl[2] + c - 1] : 0, udc = dc ? out.ucond_of_gid[bl[2] + dc - 1] : 0;
                uint64_t need = 1, need_false = 0;   // mask forms
                for (const uint32_t x : {uc, udc})
                    if (!index_form) (x & kNegated ? need_false : need) |= 1ull << (x & ~kNegated);
                uint32_t *u = urows.data() + 4 * (size_t)at++;
                u[0] = bl[0] + r;
                u[1] = (role == CB_ROLE_ANY ? 0xFFu : role) | effect << 8;
                u[2] = index_form ? (uc | udc << 8) : (uint32_t)need;
                u[3] = index_form ? 0u : out.complement ? (uint32_t)need_false : (uint32_t)(need >> 32);
                n_deny += pass == 0;
            }
        }
        ublocks[4 * b + 2] = n_deny;
        ublocks[4 * b + 3] = 0;
    }
    // Chain descriptors: one step record per RES_BLOCK_MAP entry (version, kind pattern, scope s), so that the walk
    // (cb::uc_walk) reads one record per scope instead of the block map, the block, the scope flags and the parent chain:
    //   row ranges: {first DENY row, first ALLOW row, end of the ALLOW rows, next scope of the resource chain (chain_next; CB_NONE32)}
    //   segments:   {first slot of the block's segment, ALLOW mask of the scope (~0u or 0), ~0u: the ALLOW slots hold DENY rows, else 0,
    //                next scope}
    // A scope whose ALLOWs do not count (SCOPE_PERM != 1) lists no ALLOW rows, or gets ALLOW mask 0: the walk applies a
    // scope's ALLOW mask only where they count, so those rows can never change a result.  Not lenient-dependent: only the
    // chain's first scope is (chain_start, per request).
    const uint32_t nS = meta[CB_META_N_SCOPES];
    const uint64_t n_map = (uint64_t)meta[CB_META_N_VERSIONS] * meta[CB_META_N_RESPATS] * nS;
    if (nS == 0 || len[CB_SEC_SCOPE_PARENT] < (uint64_t)nS * 4 || len[CB_SEC_SCOPE_FLAGS] < (uint64_t)nS * 4 || len[CB_SEC_RES_BLOCK_MAP] < n_map * 4) {
        out.why = "scope tables do not match the block map";
        return out;
    }
    const uint32_t *parent = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_SCOPE_PARENT]);
    const uint32_t *sflags = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_SCOPE_FLAGS]);
    const uint32_t *bmap = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_RES_BLOCK_MAP]);
    std::vector<uint32_t> next(nS);
    for (uint32_t s = 0; s < nS; s++) {
        uint32_t x = s, steps = 0;
        do { x = parent[x]; } while (x != CB_NONE32 && x < nS && ++steps <= nS && !(sflags[x] & CB_SCOPE_FLAG_RESOURCE));
        if (x != CB_NONE32 && (x >= nS || steps > nS)) { out.why = "scope parent chain out of range"; return out; }
        next[s] = x;
    }
    // Segment form: block b gets the fixed segment b + 1 of deny_rows DENY slots followed by allow_rows ALLOW slots, the
    // same counts for every block; segment 0 stays empty for scopes without a block.  The slot section names the image
    // row of every slot (the rows themselves stay as above); the library merges the rows with the batch in slot order
    // (cb::UcRowsGlobal), where a slot's position gives its effect, so the merged record drops it, and an unused slot
    // (CB_NONE32) becomes the zero record, whose action mask 0 contributes nothing.  The walk then runs a fixed number of rows per scope at constant
    // offsets from the segment base, with no per-row clamp or effect test.  Only rows the walk can use take slots: those of
    // blocks the block map names, and ALLOW rows only of blocks named from a scope whose ALLOWs count.  A block named only
    // from scopes whose ALLOWs do not count has DENY rows alone; they fill its whole segment, and its descriptors route
    // the ALLOW slots into the scope's DENY mask.  So the counts are: deny_rows, the most DENY rows of a block whose ALLOWs
    // count; allow_rows, the most ALLOW rows of such a block, or more, so that every DENY-only block fits.  Tables whose
    // segment would pass the unroll bound of the specialised walk (cb::kUcUnrollRows) keep the row ranges and their loop.
    std::vector<uint8_t> used(n_blocks, 0);   // bit 0: named by the block map; bit 1: from a scope whose ALLOWs count
    for (uint64_t e = 0; e < n_map; e++) {
        const uint32_t bid = bmap[e];
        if (bid == CB_NONE32) continue;
        if (bid >= n_blocks) { out.why = "block map entry out of range"; return out; }
        used[bid] |= 1 | (((sflags[e % nS] >> CB_SCOPE_PERM_SHIFT) & 3) == 1) << 1;
    }
    uint32_t max_deny = 0, max_allow = 0, max_deny_only = 0;
    for (uint32_t b = 0; b < n_blocks; b++) {
        const uint32_t *bl = ublocks.data() + 4 * (size_t)b;   // {row_start, n_rows, DENY rows, 0}
        if (used[b] & 2) {
            max_deny = bl[2] > max_deny ? bl[2] : max_deny;
            max_allow = bl[1] - bl[2] > max_allow ? bl[1] - bl[2] : max_allow;
        } else if (used[b]) max_deny_only = bl[2] > max_deny_only ? bl[2] : max_deny_only;
    }
    if (max_deny_only > max_deny + max_allow) max_allow = max_deny_only - max_deny;
    const uint32_t seg = max_deny + max_allow;
    const bool segments = seg >= 1 && seg <= cb::kUcUnrollRows && ((uint64_t)n_blocks + 1) * seg < (1ull << 31);
    std::vector<uint32_t> slots;   // segment form: the image row of every slot, CB_NONE32 for an unused one
    if (segments) {
        out.deny_rows = max_deny;
        out.allow_rows = max_allow;
        slots.assign(((size_t)n_blocks + 1) * seg, CB_NONE32);
        for (uint32_t b = 0; b < n_blocks; b++) {
            const uint32_t *bl = ublocks.data() + 4 * (size_t)b;
            const uint32_t n_use = (used[b] & 2) ? bl[1] : used[b] ? bl[2] : 0;
            for (uint32_t r = 0; r < n_use; r++)   // DENY-only blocks: every row in order, over both parts
                slots[(size_t)(b + 1) * seg + (r < bl[2] || !(used[b] & 2) ? r : max_deny + r - bl[2])] = bl[0] + r;
        }
    }
    std::vector<uint32_t> chain(4 * (size_t)n_map, 0);
    for (uint64_t e = 0; e < n_map; e++) {
        const uint32_t s = (uint32_t)(e % nS), bid = bmap[e];
        uint32_t *d = chain.data() + 4 * e;
        if (bid != CB_NONE32) {   // (below n_blocks: checked above)
            const uint32_t *bl = ublocks.data() + 4 * (size_t)bid;   // {row_start, n_rows, DENY rows, 0}
            const bool allow_counts = ((sflags[s] >> CB_SCOPE_PERM_SHIFT) & 3) == 1;
            if (segments) {
                d[0] = (bid + 1) * seg;
                d[1] = allow_counts ? ~0u : 0u;
                d[2] = (used[bid] & 2) ? 0u : ~0u;
            } else {
                d[0] = bl[0];
                d[1] = bl[0] + bl[2];
                d[2] = allow_counts ? bl[0] + bl[1] : d[1];
                out.scope_rows = d[2] - d[0] > out.scope_rows ? d[2] - d[0] : out.scope_rows;
            }
        }
        d[3] = next[s];
    }
    if (segments) out.scope_rows = seg;
    // read by cb_specialize.h: generate_uc (the walk's form and its unroll bounds)
    ucond_rec[0] = out.scope_rows;
    ucond_rec[1] = out.deny_rows;
    ucond_rec[2] = out.allow_rows;
    ucond_rec[3] = out.complement ? out.n_bits : 0u;
    // compact image: the sections the unique-condition kernels (and the interpreter they may call) read
    out.lay = lay;
    for (auto &o : out.lay.off) o = 0;
    auto append = [&](const void *p, uint64_t n) {
        const uint32_t at = (uint32_t)out.bytes.size();
        out.bytes.resize((out.bytes.size() + n + 15) & ~(size_t)15, 0);
        if (n) memcpy(out.bytes.data() + at, p, n);
        return at;
    };
    append("CBUC", 4);   // offset 0 stays unused: a zero offset means "section not present"
    // (the blocks and the block map are folded into the chain descriptors)
    for (int id : {CB_SEC_SCOPE_PARENT, CB_SEC_SCOPE_FLAGS, CB_SEC_CODE, CB_SEC_CONSTS, CB_SEC_CONSTS_V64, CB_SEC_THEAP,
                   CB_SEC_STR_OFF, CB_SEC_STR_BYTES})
        out.lay.off[id] = append(image + off[id], len[id]);
    out.lay.uc_conds_off = append(ucond_rec.data(), ucond_rec.size() * 4);
    out.lay.uc_rows_off = append(urows.data(), urows.size() * 4);
    out.lay.uc_chain_off = append(chain.data(), chain.size() * 4);
    out.lay.uc_slots_off = segments ? append(slots.data(), slots.size() * 4) : 0;
    out.lay.n_uconds = out.n_bits;
    out.lay.uc_complement = out.complement;
    out.lay.uc_n_rows = segments ? (uint32_t)slots.size() : (uint32_t)(urows.size() / 4);
    out.lay.uc_deny_rows = out.deny_rows;
    out.lay.uc_allow_rows = out.allow_rows;
    out.lay.theap_words = (uint32_t)(len[CB_SEC_THEAP] / 8);
    out.lay.image_bytes = (uint32_t)out.bytes.size();
    out.ok = true;
    return out;
}

// Side table of the metadata kernels (cb::eval_request_uc_meta), kept apart from the image so that the effect kernels read
// the same bytes as without it.  16-byte records:
//   one per RES_BLOCK_MAP entry (version, kind pattern, scope s), indexed like the chain descriptors:
//     {first derived-role record, end, bit 0: a resource policy of this kind exists from s to the end of the chain |
//      scope levels from s to the end of the chain << 8 (saturating at CB_MAX_CHAIN + 1), 0}
//   then the derived roles of every block the map names (DR_OFF / DR_ENTRIES / DR_PARENTS, in block order):
//     {name bit, condition bit (cond_bit; 0: none) | it must be clear (complement-coded image) << 30 | any parent role << 31,
//      parent-role mask over the table roles (lo, hi)}
// Only for the tables the unique-condition kernels take whose metadata needs nothing but the resource chain: no principal
// or role policies, no parent roles (so a parent role matches a request role by equality, cb::role_in_pr), no condition
// reading runtime.effectiveDerivedRoles, and no principal-policy existence bits.
struct MetaSide {
    bool ok = false;
    std::string why;                // when !ok
    std::vector<uint32_t> words;    // 4 per record
};

inline MetaSide build_meta(const uint8_t *image, const uint32_t *off, const uint64_t *len, const uint32_t *meta, const cb::TableLayout &lay, const Image &uc) {
    MetaSide out;
    if (!uc.ok) { out.why = "no unique-condition image"; return out; }
    if (lay.has_principal_policies || lay.has_role_policies || lay.has_parent_roles || lay.uses_runtime) {
        out.why = "principal / role policies, parent roles or runtime.effectiveDerivedRoles";
        return out;
    }
    const uint32_t nS = lay.nS, n_blocks = meta[CB_META_N_BLOCKS];
    const uint64_t n_map = (uint64_t)lay.nV * lay.nRP * nS;
    const uint8_t *pex = image + off[CB_SEC_PRIN_EXISTS];
    for (uint64_t i = 0; i < (uint64_t)lay.nV * nS; i++)
        if (pex[i]) { out.why = "principal-policy existence bits"; return out; }
    const uint32_t *bmap = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_RES_BLOCK_MAP]);
    const uint8_t *rex = image + off[CB_SEC_RES_EXISTS];
    const uint32_t *dr_off = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_DR_OFF]);
    const uint32_t *dr_ent = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_DR_ENTRIES]);
    const uint32_t *dr_par = reinterpret_cast<const uint32_t *>(image + off[CB_SEC_DR_PARENTS]);
    const uint64_t n_ent = len[CB_SEC_DR_ENTRIES] / 16, n_par = len[CB_SEC_DR_PARENTS] / 4;
    const uint32_t *chain = reinterpret_cast<const uint32_t *>(uc.bytes.data() + uc.lay.uc_chain_off);   // {.., .., .., next scope}
    // scope levels from s to the end of the resource chain
    std::vector<uint32_t> levels(nS, 0);
    for (uint32_t s = 0; s < nS; s++) {
        uint32_t n = 0;
        for (uint32_t x = s; x != CB_NONE32 && n <= CB_MAX_CHAIN; x = chain[4 * (uint64_t)x + 3]) n++;
        levels[s] = n;
    }
    out.words.assign(4 * n_map, 0);
    std::vector<uint32_t> first(n_blocks, CB_NONE32), end(n_blocks, 0);   // derived-role records of a block, once emitted
    for (uint64_t e = 0; e < n_map; e++) {
        const uint32_t s = (uint32_t)(e % nS), bid = bmap[e];
        uint32_t exists = 0;
        for (uint32_t x = s, n = 0; x != CB_NONE32 && n <= CB_MAX_CHAIN; x = chain[4 * (e - s + x) + 3], n++) exists |= rex[e - s + x] & CB_EXISTS_RESOURCE_KIND;
        out.words[4 * e + 2] = (exists ? 1u : 0u) | levels[s] << 8;
        if (bid == CB_NONE32) continue;   // (below n_blocks: cbuc::build checked the map)
        if (first[bid] == CB_NONE32) {
            first[bid] = (uint32_t)(out.words.size() / 4);
            if (dr_off[bid] > dr_off[bid + 1] || dr_off[bid + 1] > n_ent) { out.why = "derived-role range out of range"; return out; }
            for (uint32_t j = dr_off[bid]; j < dr_off[bid + 1]; j++) {
                const uint32_t *en = dr_ent + 4 * (uint64_t)j;   // {name index, cond + 1, parents start, n parents}
                if ((uint64_t)en[2] + en[3] > n_par || (en[1] && en[1] - 1 >= uc.ucond_of_gid.size())) { out.why = "derived-role entry out of range"; return out; }
                uint64_t mask = 0;
                bool any = false;
                for (uint32_t q = 0; q < en[3]; q++) {
                    const uint32_t pr = dr_par[en[2] + q];
                    if (pr == CB_ROLE_ANY) any = true;
                    else if (pr < lay.nR) mask |= 1ull << pr;   // (nR <= 64: cbuc::build)
                }
                const uint32_t u = en[1] ? uc.ucond_of_gid[en[1] - 1] : 0u;
                out.words.insert(out.words.end(), {en[0] & 63u, (u & ~kNegated) | (u & kNegated ? 1u << 30 : 0u) | (any ? 1u << 31 : 0u),
                                                   (uint32_t)mask, (uint32_t)(mask >> 32)});
            }
            end[bid] = (uint32_t)(out.words.size() / 4);
        }
        out.words[4 * e] = first[bid];
        out.words[4 * e + 1] = end[bid];
    }
    out.ok = true;
    return out;
}

}  // namespace cbuc
