// raft_step.cuh -- the device logic, compiled twice:
//   ra_wide    every index / term is 64 bits wide (the ABI's width): the general kernel, the wide hot kernel, the
//              host emulation
//   ra_narrow  the hot kernel's fast paths on 32-bit arithmetic, for rows all of whose values fit (see
//              raft_logic.cuh "narrow pass"): same source, `ix_t` = u32
// Everything else in the engine sees the wide names.
#pragma once
#include "raft_common.cuh"

#define RA_NARROW_PASS 0
namespace ra_wide {
#include "raft_logic.cuh"
#include "raft_row_logic.cuh"
}
#undef RA_NARROW_PASS
#define RA_NARROW_PASS 1
namespace ra_narrow {
#include "raft_logic.cuh"
#include "raft_row_logic.cuh"
}
#undef RA_NARROW_PASS
using namespace ra_wide;
