// Argument checks of the host-pointer verify entry points that a multi-device context (hs_multi.cpp) splits across its members.
// The single-context entry points in hs_engine.cu and the hs_multi_* forms call the same check, so both reject exactly the same
// calls before anything runs.  Each returns nullptr when the arguments are valid, else the reason the entry point reports after its
// own name ("<entry point>: <reason>") with HS_ERR_ARG.
#ifndef HS_ARGS_H
#define HS_ARGS_H
#include <stddef.h>
#include <stdint.h>

#include "../../include/hs_crypto.h"

namespace hs_args {
const char *rec128(const hs_rec128 *recs, size_t n, uint32_t mode, const uint32_t *out_bitmap);
const char *msgs(const uint8_t *sig, const uint8_t *pk, const uint32_t *vidx, const uint8_t *msgs, size_t msg_len, size_t n, uint32_t mode,
                 const uint32_t *out_bitmap);
const char *groups(const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig, const uint8_t *pk, const uint32_t *vidx,
                   const uint32_t *msg_idx, const uint32_t *group_idx, const uint8_t *mode, size_t n_items, size_t n_groups,
                   const uint32_t *out_group_bitmap);
}  // namespace hs_args
#endif
