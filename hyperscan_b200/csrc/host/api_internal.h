/* api_internal.h -- shared between the host-only and CUDA halves of the ABI. */
#ifndef HSB200_API_INTERNAL_H
#define HSB200_API_INTERNAL_H

#include "../../../include/hs_b200.h"
#include "../ref_layout.h"
#include "hwlm_build.h"

namespace hsb {

extern hs_alloc_t g_db_alloc, g_misc_alloc, g_scratch_alloc, g_stream_alloc;
extern hs_free_t g_db_free, g_misc_free, g_scratch_free, g_stream_free;

hs_error_t checkAlloc(const void *p);

static inline const RoseEngine *dbRose(const hs_database_t *db) {
    const DbHeader *h = (const DbHeader *)db;
    return (const RoseEngine *)((const char *)h + h->bytecode);
}

/** Apply the process-wide build tunables set through hs_b200_set_build_option
 * (the analogue of the reference's Grey overrides, src/grey.cpp:40-160). */
void applyBuildOptions(HwlmBuildOpts *o);
int outfixEngineOption(); /* build option "outfix_engine" (api_host.cpp) */
int regexDfaOption();     /* build option "regex_dfa" (api_host.cpp) */
int mixedRoseOption();    /* build option "mixed_rose" (api_host.cpp) */

} // namespace hsb
#endif
