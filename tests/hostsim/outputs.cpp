// tests/hostsim/outputs.cpp -- DEBUG AID (test infrastructure, never shipped, never timed).
// Host build of the rule-output walk (cb::eval_request_outputs), the body check_outputs_kernel runs per request, so that
// tests/test_rule_outputs.py can hold it against oracle #1 without a GPU.  Built by tests/hostsim/outputs.py.
#include <cstdint>
#include <cstring>

#include "cb_core.h"
#include "cb_host.h"

// effects / action_meta / req_meta as cgpu_check_meta; records: n * stride bytes.  Returns 0, -1 on a bad blob or batch, or
// the status bits of the walk (1 unsupported value, cb::CB_OUT_STATUS_OVERFLOW, cb::CB_OUT_STATUS_UNLOWERED) negated.
extern "C" int hostsim_check_outputs(const void *blob, uint64_t blob_len, uint64_t n, uint32_t max_actions, int64_t now, uint32_t flags,
                                     const void *const *cols, const uint64_t *col_bytes, uint8_t *effects, uint32_t *action_meta,
                                     cb_request_meta *req_meta, uint8_t *records, uint32_t stride) {
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
    for (uint64_t i = 0; i < n; i++)
        cb::eval_request_outputs(static_cast<const uint8_t *>(blob), &lay, &b, i, effects, action_meta, req_meta, &status, records + i * stride, stride);
    return status ? -(int)(status << 1) : 0;
}
