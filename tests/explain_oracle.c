/*
 * explain_oracle.c — CPU checker of explained placement decisions (simon_explain_set, include/simon_gpu.h).  TEST INFRASTRUCTURE
 * ONLY, like the oracle it is built on.
 *
 * The CPU oracle (oracle/simon_oracle.c) is compiled into this library unchanged.  Its per-node detail of the last scheduled pod
 * (simon_oracle_last_detail: filter stage and the ten score words) names the failing stage of each node, not every reason its
 * verdict carries; this exports those reasons (the bitmask of simon_fail_code the oracle's filter stage builds for each node).
 */
#include "../oracle/simon_oracle.c"

/* The filter verdict of every node for the last pod that reached the scheduler: 0 feasible, else a bitmask of simon_fail_code. */
void simon_oracle_last_reasons(simon_oracle *o, uint32_t *out) { memcpy(out, o->reasons, 4ull * o->N); }
