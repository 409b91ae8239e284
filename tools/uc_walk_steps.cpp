// tools/uc_walk_steps.cpp -- host helper of tools/uc_walk_steps.py (built by it with g++, never shipped).
// The rows the unique-condition walk (cb::uc_walk) visits per request and scope level, from the image's chain
// descriptors (segment form: the used slots of the scope's segment): out[(i * levels + level) * 2 + {0, 1}] = DENY rows,
// ALLOW rows that count; zero past the end of the chain
// and for a request the walk does not reach.  The walk also stops once every pair of the request is decided, which
// needs the condition word: not modelled.
#include <cstdint>
#include <cstring>

#include "cb_core.h"
#include "cb_uc.h"
#include "cb_host.h"

// -> the table's longest scope, or < 0 (-1: the library would refuse the blob or the batch; -3: no unique-condition image)
extern "C" int64_t uc_walk_rows(const void *blob, uint64_t blob_len, uint64_t n, uint32_t max_actions, uint32_t flags,
                                const void *const *cols, const uint64_t *col_bytes, uint32_t levels, uint16_t *out) {
    cb::TableLayout lay;
    uint32_t meta[CB_META_WORDS];
    uint64_t sec_len[cbhost::kMaxSec] = {};
    if (!cbhost::parse_blob(blob, blob_len, &lay, meta, sec_len).empty()) return -1;
    cgpu_batch batch;
    batch.n_requests = n; batch.max_actions = max_actions; batch.now_unix_nanos = 0; batch.flags = flags;
    batch.columns = cols; batch.column_bytes = col_bytes; batch.n_columns = CGPU_N_COLUMNS;
    cb::BatchView b;
    if (!cbhost::make_batch_view(lay, &batch, 0, n, &b).empty()) return -1;
    const cbuc::Image uc = cbuc::build(static_cast<const uint8_t *>(blob), lay.off, sec_len, meta, lay);
    if (!uc.ok) return -3;
    cb::TableView ut;
    ut.base = uc.bytes.data(); ut.L = &uc.lay;
    memset(out, 0, n * levels * 2 * sizeof(uint16_t));
    for (uint64_t i = 0; i < n; i++) {   // which requests reach the walk: cb::eval_request_uc
        cb::CachedCols gc; gc.b = &b; gc.n = i;
        const cb::U4 h0 = gc.hdr0();
        const uint64_t h1 = gc.hdr1();
        const uint32_t rv = (uint32_t)(h1 & 0xFFFF), pv = (uint32_t)((h1 >> 16) & 0xFFFF), aset = (uint32_t)(h1 >> 32);
        uint32_t n_roles = 0;
        for (uint32_t q = 0; q < b.role_cols; q++) n_roles = gc.role(q) != CB_ROLE_PAD ? q + 1 : n_roles;
        const uint32_t K = aset < b.n_asets ? gc.aset_k(aset) : 0;
        if (pv != rv || n_roles == 0 || K == 0 || rv == CB_NONE16 || h0.y == CB_KIND_NONE) continue;
        const cb::U4 *chain = ut.uc_chain() + (rv * uc.lay.nRP + h0.y) * uc.lay.nS;
        uint32_t lv = 0;
        for (uint32_t sc = cb::chain_start(ut, h0.z, CB_SCOPE_FLAG_RESOURCE, (b.flags & CB_BATCH_FLAG_LENIENT) != 0); sc != CB_NONE32 && lv < levels;
             sc = chain[sc].w, lv++) {
            const cb::U4 d = chain[sc];
            uint32_t n_deny = d.y - d.x, n_allow = d.z - d.y;
            if (uc.deny_rows + uc.allow_rows) {   // segment form: the used slots (an unused one has no original row)
                n_deny = n_allow = 0;
                for (uint32_t j = 0; j < uc.deny_rows + uc.allow_rows; j++)
                    if (ut.uc_slots()[d.x + j] != CB_NONE32) (j < uc.deny_rows || d.z ? n_deny : n_allow)++;
                n_allow = d.y ? n_allow : 0;
            }
            out[(i * levels + lv) * 2] = (uint16_t)n_deny;
            out[(i * levels + lv) * 2 + 1] = (uint16_t)n_allow;
        }
    }
    return uc.scope_rows;   // segment form: the slots every scope runs
}
