// TEST INFRASTRUCTURE: kta_push over numpy columns, one call per record, from C (feed.push_records loads it with ctypes).
// A Python loop spends microseconds per record around the call; this one spends what the caller of kta_push would.
// Host code only.  kta_push is passed in as a function pointer, so the loop calls whichever build of the library the
// test process loaded.
#include <cstdint>

#include "../../include/kta.h"

using push_fn = decltype(&kta_push);

// Records [0, n): record i's key is key_len[i] bytes at keys + key_off[i] (NULL when key_len[i] <= 0).  Returns 0, or the
// first failing call's status with *failed set to its record.
extern "C" int push_loop(push_fn push, kta_handle *h, int64_t n, const int32_t *partition, const int64_t *offset,
                         const int64_t *ts_ms, const int32_t *key_len, const int32_t *value_len, const uint8_t *keys,
                         const int64_t *key_off, int64_t *failed) {
    for (int64_t i = 0; i < n; i++) {
        const int rc = push(h, partition[i], offset[i], ts_ms[i], key_len[i] > 0 ? keys + key_off[i] : nullptr, key_len[i],
                            value_len[i]);
        if (rc) {
            *failed = i;
            return rc;
        }
    }
    return 0;
}
