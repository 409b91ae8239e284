// tests/hostsim/hostsim.cpp -- DEBUG AID (test infrastructure, never shipped, never timed).
// Compiles the kernels' per-request core (cerbos_b200/csrc/cb_core.h) for the host so its logic can be
// checked against the oracles on a machine without a GPU.  The product
// library (libcerbos_b200.so) contains no such path: without a CUDA device cgpu_init fails.
#include <cstdint>
#include <cstring>
#include <vector>

#include "cb_core.h"
#include "cb_specialize.h"
#include "cb_uc.h"
#include "cb_encode.h"
#include "cb_host.h"

#if defined(HOSTSIM_SPEC_UC)
#include "spec_gen.inc"   // generated for one table by hostsim_generate_uc: cb::SpecConds (unique-condition form)
typedef cb::GenericBlocks HostBlocks;
typedef cb::SpecConds HostConds;
#define HOSTSIM_ENTRY hostsim_check_spec
#elif defined(HOSTSIM_SPEC)
#include "spec_gen.inc"   // generated for one table by hostsim_generate (tests/test_specialize.py)
typedef cb::SpecBlocks HostBlocks;
typedef cb::GenericConds HostConds;
#define HOSTSIM_ENTRY hostsim_check_spec
#else
typedef cb::GenericBlocks HostBlocks;
typedef cb::GenericConds HostConds;
#define HOSTSIM_ENTRY hostsim_check
#endif

extern "C" {
uint64_t hostsim_deferred = 0;   // requests the lean / unique-condition body left to the general body in the last call
int hostsim_body = 1;            // the body the last check call ran, by the mode that selects it (1: the general 64-bit body)
}

// A table and a batch set up the way the library sets them up (cb_host.h)
struct Setup {
    const uint8_t *base = nullptr;
    cb::TableLayout lay;
    uint32_t meta[CB_META_WORDS];
    uint64_t sec_len[cbhost::kMaxSec] = {};
    cb::BatchView b;
};
// false: the library would refuse the blob, or (cols given) the batch
static bool setup(Setup &s, const void *blob, uint64_t blob_len, const void *const *cols = nullptr, const uint64_t *col_bytes = nullptr,
                  uint64_t n = 0, uint32_t max_actions = 0, int64_t now = 0, uint32_t flags = 0) {
    s.base = static_cast<const uint8_t *>(blob);
    if (!cbhost::parse_blob(blob, blob_len, &s.lay, s.meta, s.sec_len).empty()) return false;
    if (!cols) return true;
    cgpu_batch batch;
    batch.n_requests = n; batch.max_actions = max_actions; batch.now_unix_nanos = now; batch.flags = flags;
    batch.columns = cols; batch.column_bytes = col_bytes; batch.n_columns = CGPU_N_COLUMNS;
    return cbhost::make_batch_view(s.lay, &batch, 0, n, &s.b).empty();
}

extern "C" int HOSTSIM_ENTRY(const void *blob, uint64_t blob_len, uint64_t n, uint32_t max_actions, int64_t now, uint32_t flags,
                             const void *const *cols, const uint64_t *col_bytes, uint8_t *bitmap, int mode) {
    Setup s;
    if (!setup(s, blob, blob_len, cols, col_bytes, n, max_actions, now, flags)) return -1;
    cb::BatchView &b = s.b;
    const cb::TableLayout &lay = s.lay;
    cb::TableView t;
    t.base = s.base; t.L = &lay;
    uint32_t status = 0;
    hostsim_deferred = 0;
    hostsim_body = 1;
    // mode 0: the lean body reading the columns from global memory (the library's lean kernel; it gives tables whose blocks
    // differ in shape to the unique-condition kernel, modes 4 / 5, instead); 1: force the general 64-bit body; 2: general
    // 32-bit body; 3: the lean body reading a tile of the columns staged the way the kernel's TMA copies lay it out in shared
    // memory.  A mode the table or batch cannot take runs the general 64-bit body.
    const bool lean = cbhost::lean_eligible(lay, s.meta, b);
    // modes 4 / 5: the unique-condition body (cb_uc.h image) with rows read from the image / from merged 8-byte records
    if ((mode == 4 || mode == 5) && lean) {
        const cbuc::Image uc = cbuc::build(s.base, lay.off, s.sec_len, s.meta, lay);
        if (!uc.ok) return -3;
        if (cbhost::uc_eligible(lay, uc, b)) {
            hostsim_body = mode;
            cb::TableView ut;
            ut.base = uc.bytes.data(); ut.L = &uc.lay;
            std::vector<cb::U4> pk((size_t)b.n_asets * b.n_rows);
            for (size_t j = 0; j < pk.size(); j++) {
                const cb::U4 u = ut.urows()[j % b.n_rows];
                pk[j] = cb::uc_row_record(u, (uint32_t)b.row_am[(j / b.n_rows) * b.n_rows + u.x], b.rcp, lay.nR);
            }
#if defined(HOSTSIM_SPEC_UC)
            // the per-string predicate words the library's pre-pass kernel would compute (one per table / batch string)
            std::vector<uint32_t> strpred(lay.nT + b.n_bstr + 1, 0);
            if (HostConds::n_strpred)
                for (uint32_t id = 0; id < lay.nT + b.n_bstr; id++) strpred[id] = HostConds().strpred(ut, b, id);
            b.strpred = strpred.data();
#endif
            for (uint64_t i = 0; i < n; i++) {
                cb::CachedCols gc; gc.b = &b; gc.n = i;
                bool d;
                if (mode == 5) { cb::UcRowsPacked rows; rows.pk = pk.data(); d = cb::eval_request_uc(ut, b, gc, rows, i, bitmap, nullptr, HostConds()); }
                else { cb::UcRowsGlobal rows; rows.urows = ut.urows(); rows.row_am = b.row_am; rows.RCP = b.rcp; rows.nR = lay.nR; d = cb::eval_request_uc(ut, b, gc, rows, i, bitmap, nullptr, HostConds()); }
                if (d) { hostsim_deferred++; cb::eval_request_general(t.base, t.L, &b, i, bitmap, nullptr, &status); }
            }
            return status ? -2 : 0;
        }
    }
    if (mode == 3 && lean) {
        hostsim_body = 3;
        std::vector<uint64_t> tile(cb::tile_cols_bytes(b.role_cols, lay.n_slots) / 8 + 2);
        uint8_t *tb = reinterpret_cast<uint8_t *>(tile.data());
        for (uint64_t t0 = 0; t0 < n; t0 += cb::CB_TILE) {
            const uint64_t cnt = n - t0 < cb::CB_TILE ? n - t0 : cb::CB_TILE;
            memcpy(tb, b.hdr0 + t0, cnt * 16);
            memcpy(tb + cb::CB_TILE * 16, b.hdr1 + t0, cnt * 8);
            for (uint32_t i = 0; i < b.role_cols; i++) memcpy(tb + cb::CB_TILE * 24 + i * cb::CB_TILE * 4, b.roles + i * b.stride + t0, cnt * 4);
            const uint32_t so = cb::CB_TILE * (24 + 4 * b.role_cols);
            for (uint32_t v = 0; v < lay.n_slots; v++) memcpy(tb + so + v * cb::CB_TILE * 8, b.slots + v * b.stride + t0, cnt * 8);
            for (uint32_t j = 0; j < cnt; j++) {
                cb::TileCols tc; tc.base = tb; tc.tid = j; tc.slots_off = so; tc.aset_k_s = b.aset_k; tc.row_am_s = b.row_am; tc.res_s = nullptr;
                if (cb::eval_request_fast(t, b, tc, t0 + j, bitmap, nullptr, HostBlocks())) cb::eval_request_general(t.base, t.L, &b, t0 + j, bitmap, nullptr, &status);
            }
        }
        return status ? -2 : 0;
    }
    const bool narrow = b.n_pass == 1 && (uint64_t)b.max_actions * b.role_cols <= 32;
    if ((mode == 0 && lean) || (mode == 2 && narrow)) hostsim_body = mode;
    for (uint64_t i = 0; i < n; i++) {
        if (mode == 0 && lean) {
            cb::GlobalCols gc; gc.b = &b; gc.n = i;
            if (cb::eval_request_fast(t, b, gc, i, bitmap, nullptr, HostBlocks())) cb::eval_request_general(t.base, t.L, &b, i, bitmap, nullptr, &status);
        }
        else if (mode == 2 && narrow) cb::eval_request<uint32_t>(t, b, i, bitmap, nullptr, &status);
        else cb::eval_request<uint64_t>(t, b, i, bitmap, nullptr, &status);
    }
    return status ? -2 : 0;
}

#if !defined(HOSTSIM_SPEC) && !defined(HOSTSIM_SPEC_UC)
// the native batch encoder (cb_encode.h): n serialized CheckInput messages -> the twelve columns; the caller reads them
// back through hostsim_encoded_column() and releases with hostsim_encoded_free()
struct HostEncoded { cbenc::Columns cols; };
extern "C" void *hostsim_encode(const void *blob, uint64_t blob_len, const char *default_version, const char *default_scope, int lenient,
                                const void *const *inputs, const uint64_t *lens, uint64_t n, uint32_t *dims /* max_actions, role_cols, kc, n_pass */, uint32_t n_threads) {
    cbenc::Encoder enc;
    cbenc::Conf conf;
    conf.default_version = default_version; conf.default_scope = default_scope; conf.lenient = lenient != 0;
    if (!enc.init(blob, blob_len, conf)) return nullptr;
    std::vector<size_t> ls(lens, lens + n);
    HostEncoded *he = new HostEncoded();
    if (!enc.encode(inputs, ls.data(), n, &he->cols, n_threads)) { delete he; return nullptr; }
    dims[0] = he->cols.max_actions; dims[1] = he->cols.role_cols; dims[2] = he->cols.kc; dims[3] = he->cols.n_pass;
    return he;
}
extern "C" const void *hostsim_encoded_column(const void *h, int i, uint64_t *bytes) {
    const HostEncoded *he = static_cast<const HostEncoded *>(h);
    *bytes = he->cols.bytes(i);
    return he->cols.ptr(i);
}
extern "C" void hostsim_encoded_free(void *h) { delete static_cast<HostEncoded *>(h); }

// the decision-metadata body (cb::eval_request_meta): effects + per-action metadata words + per-request metadata
extern "C" int hostsim_check_meta(const void *blob, uint64_t blob_len, uint64_t n, uint32_t max_actions, int64_t now, uint32_t flags,
                                  const void *const *cols, const uint64_t *col_bytes, uint8_t *effects, uint32_t *action_meta, cb_request_meta *req_meta) {
    Setup s;
    if (!setup(s, blob, blob_len, cols, col_bytes, n, max_actions, now, flags)) return -1;
    uint32_t status = 0;
    for (uint64_t i = 0; i < n; i++) cb::eval_request_meta(s.base, &s.lay, &s.b, i, effects, action_meta, req_meta, &status);
    return status ? -2 : 0;
}
// the unique-condition form of the specialised source (cb::SpecConds); "" if the table does not qualify; *n_uconds_out = distinct conditions
extern "C" int64_t hostsim_generate_uc(const void *blob, uint64_t blob_len, char *out, uint64_t cap, uint32_t *n_uconds_out) {
    Setup s;
    if (!setup(s, blob, blob_len)) return -1;
    const cbuc::Image uc = cbuc::build(s.base, s.lay.off, s.sec_len, s.meta, s.lay);
    if (n_uconds_out) *n_uconds_out = uc.ok ? uc.n_uconds : 0;
    std::string src = uc.ok ? cbspec::generate_uc(uc.bytes.data(), uc.lay.off, uc.lay.uc_conds_off, uc.n_uconds, s.lay.n_slots, s.meta[CB_META_N_CONSTS]).src : std::string();
    if (src.size() + 1 > cap) return -(int64_t)src.size() - 2;
    memcpy(out, src.c_str(), src.size() + 1);
    return (int64_t)src.size();
}
// the table-specialised block evaluators the library would hand to NVRTC (source text; "" if the table does not qualify)
extern "C" int64_t hostsim_generate(const void *blob, uint64_t blob_len, char *out, uint64_t cap) {
    Setup s;
    if (!setup(s, blob, blob_len)) return -1;
    std::string src = cbspec::generate(s.base, s.lay.off, s.meta);
    if (src.size() + 1 > cap) return -(int64_t)src.size() - 2;
    memcpy(out, src.c_str(), src.size() + 1);
    return (int64_t)src.size();
}
#endif
