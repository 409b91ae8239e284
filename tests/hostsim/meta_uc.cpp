// tests/hostsim/meta_uc.cpp -- DEBUG AID (test infrastructure, never shipped, never timed).
// Host build of the metadata form of the unique-condition body (cb::eval_request_uc_meta) next to the reference-order
// metadata body (cb::eval_request_meta), so that tests/test_meta_uc.py can hold the two against each other without a GPU.
// Built plain (generic conditions, cb::GenericConds) or, with HOSTSIM_SPEC_UC, with the conditions generated for one table
// (spec_gen.inc: cb::SpecConds), by tests/hostsim/meta_uc.py.
#include <cstdint>
#include <cstring>
#include <vector>

#include "cb_core.h"
#include "cb_specialize.h"
#include "cb_uc.h"
#include "cb_host.h"

#if defined(HOSTSIM_SPEC_UC)
#include "spec_gen.inc"   // generated for one table by hostsim_generate_uc (tests/hostsim/hostsim.cpp)
typedef cb::SpecConds HostConds;
#else
typedef cb::GenericConds HostConds;
#endif

extern "C" {
uint64_t meta_uc_deferred = 0;   // requests the unique-condition metadata body left to the reference-order body in the last call
int meta_uc_took = 0;            // whether the last call ran the unique-condition metadata body at all
}

// The arguments of hostsim_check_meta: the three planes from cb::eval_request_uc_meta, its deferred requests through
// cb::eval_request_meta; the whole batch through the latter when the table or batch does not qualify (as the library
// decides: lean and unique-condition eligible, and a metadata side table).
extern "C" int hostsim_check_meta_uc(const void *blob, uint64_t blob_len, uint64_t n, uint32_t max_actions, int64_t now, uint32_t flags,
                                     const void *const *cols, const uint64_t *col_bytes, uint8_t *effects, uint32_t *action_meta, cb_request_meta *req_meta) {
    const uint8_t *base = static_cast<const uint8_t *>(blob);
    cb::TableLayout lay;
    uint32_t meta[CB_META_WORDS];
    uint64_t sec_len[cbhost::kMaxSec] = {};
    if (!cbhost::parse_blob(blob, blob_len, &lay, meta, sec_len).empty()) return -1;
    cgpu_batch batch;
    batch.n_requests = n; batch.max_actions = max_actions; batch.now_unix_nanos = now; batch.flags = flags;
    batch.columns = cols; batch.column_bytes = col_bytes; batch.n_columns = CGPU_N_COLUMNS;
    cb::BatchView b;
    if (!cbhost::make_batch_view(lay, &batch, 0, n, &b).empty()) return -1;
    uint32_t status = 0;
    meta_uc_deferred = 0;
    const cbuc::Image uc = cbuc::build(base, lay.off, sec_len, meta, lay);
    const cbuc::MetaSide side = cbuc::build_meta(base, lay.off, sec_len, meta, lay, uc);
    const bool take = cbhost::lean_eligible(lay, meta, b) && cbhost::uc_eligible(lay, uc, b) && side.ok;
    meta_uc_took = take;
    cb::TableView ut;
    ut.base = uc.bytes.data(); ut.L = &uc.lay;
#if defined(HOSTSIM_SPEC_UC)
    // the per-string predicate words the library's pre-pass kernel would compute (one per table / batch string)
    std::vector<uint32_t> strpred(lay.nT + b.n_bstr + 1, 0);
    if (take && HostConds::n_strpred)
        for (uint32_t id = 0; id < lay.nT + b.n_bstr; id++) strpred[id] = HostConds().strpred(ut, b, id);
    b.strpred = strpred.data();
#endif
    const cb::U4 *sp = reinterpret_cast<const cb::U4 *>(side.words.data());
    for (uint64_t i = 0; i < n; i++) {
        if (take) {
            cb::CachedCols gc; gc.b = &b; gc.n = i;
            cb::UcRowsGlobal rows; rows.urows = ut.urows(); rows.row_am = b.row_am; rows.RCP = b.rcp; rows.nR = lay.nR;
            if (!cb::eval_request_uc_meta(ut, b, gc, rows, sp, i, effects, action_meta, req_meta, HostConds())) continue;
            meta_uc_deferred++;
        }
        cb::eval_request_meta(base, &lay, &b, i, effects, action_meta, req_meta, &status);
    }
    return status ? -2 : 0;
}
