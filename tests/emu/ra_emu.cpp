/* TEST INFRASTRUCTURE -- not part of the product, never loaded by ra_b200/.
 *
 * Host emulation of the engine's two step kernels: the DEVICE LOGIC headers of the product
 * (ra_b200/csrc/raft_step.cuh, raft_row.cuh -- fast_event, process_event, emit_msg, the record
 * head/tail codec, row_end_of_step, load_row / read_row ...) are compiled here as plain C++
 * through tests/emu/cuda_shim.h and driven one row at a time with the control flow of
 * raft_step_kernel (fast paths until a row stalls) and raft_general_kernel (resume from the
 * 64-byte stall context).  Of the hot kernel's TMA fetch it models what a row can see: how many
 * chunks of a record tile the size flags let through (the rest reads as poison, see tile_sizes).
 * What is NOT covered is the rest of the kernels' own frame in engine.cu (the TMA ring itself,
 * warp reductions, launch plumbing): that is what the `-m gpu` tests are for.  The point of this
 * library is that the CPU test tier diffs the very source the GPU runs against the oracle
 * (tests/test_emu_parity.py), so a logic regression shows up before any GPU time is spent.
 *
 * The C ABI of include/ra_engine.h under the header's names, so that the product's host-side callers
 * (host_flood.cu, the dirty-NIF shim) link against it; only the emulation's own calls are ra_emu_*.
 * Shards: the bucket transport (ra_engine_set_outbox / ra_engine_deliver) and the peer transport
 * (ra_engine_peer_get / ra_engine_peer_set: the step stores straight into the other shards' mailbox
 * planes and count bytes).  The shards of
 * one process step one after another and share the buffer parity `cur`, so a shard's stores into
 * another's `cur ^ 1` buffer stay invisible to that shard's step: the lock step of the GPU transport.
 */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>
#include <new>
#include "cuda_shim.h"
#include "../../ra_b200/csrc/raft_step.cuh"
#include "../../ra_b200/csrc/raft_row.cuh"

struct ra_engine {
    ra_engine_cfg cfg;
    Cols C;
    int cur;
    u64 step_no, steps;
    void* allocs[96]; int n_allocs;
    int narrow, narrow_mode;                          // as engine.cu: RA_STEP_WIDE unset = auto, 0 = always narrow, 1 = never
    int out_pending;                                  // a step's outputs did not fit: they wait in the row slots
    // the split phase (ra_engine_submit / ra_engine_collect): up to two calls in flight, oldest first.  The emulation
    // evaluates a call when it is submitted and hands its result over at collect.
    struct { int rc; size_t nm, nn; } sub[2];
    int sub_n;
    int sub_abort;                                    // != 0: the status a call submitted now gets without being
                                                      // evaluated (a call in flight was rejected, or its outputs did not
                                                      // fit: RA_E_PENDING); cleared once no call is in flight
    int out_held;                                     // the call whose outputs did not fit is still in flight
};

template <typename T>
static int halloc(ra_engine* e, T** p, size_t count)
{
    void* q = calloc(count ? count : 1, sizeof(T));
    if (!q) return RA_E_NOMEM;
    e->allocs[e->n_allocs++] = q;
    *p = (T*)q;
    return RA_OK;
}

extern "C" void ra_engine_destroy(ra_engine* e)
{
    if (!e) return;
    for (int i = 0; i < e->n_allocs; i++) free(e->allocs[i]);
    free(e);
}

extern "C" int ra_engine_reset_empty(ra_engine* e)
{
    if (!e) return RA_E_INVAL;
    for (u32 r = 0; r < e->C.rows; r++) reset_row(e->C, r);
    memset(e->C.counters, 0, RA_N_COUNTERS * sizeof(u64));
    e->C.q_used[0] = 0;
    e->cur = 0; e->step_no = 0; e->steps = 0;
    e->narrow = e->narrow_mode != 2;
    e->out_pending = 0; e->sub_n = 0; e->sub_abort = 0; e->out_held = 0;   // as the engine drops its calls in flight
    return RA_OK;
}

extern "C" int ra_engine_create(const ra_engine_cfg* cfg, ra_engine** out)
{
    ra_engine_cfg c;
    int narrow_mode;
    if (!out || cfg_resolve(cfg, c, narrow_mode) != RA_OK) return RA_E_INVAL;
    ra_engine* e = (ra_engine*)calloc(1, sizeof(ra_engine));
    if (!e) return RA_E_NOMEM;
    e->cfg = c;
    e->narrow_mode = narrow_mode;
    int rc = cols_init(e->C, e->cfg, [e](auto*& p, size_t n) { return halloc(e, &p, n); });
    if (rc == RA_OK) rc = ra_engine_reset_empty(e);
    if (rc != RA_OK) { ra_engine_destroy(e); return rc; }
    *out = e;
    return RA_OK;
}

extern "C" int ra_engine_get_cfg(ra_engine* e, ra_engine_cfg* out)
{
    if (!e || !out) return RA_E_INVAL;
    *out = e->cfg;
    return RA_OK;
}

extern "C" int ra_engine_load_rows(ra_engine* e, const ra_row_state* rows, size_t n)
{
    const int rc = e ? load_rows_check(e->C, rows, n, e->narrow_mode, e->narrow) : RA_E_INVAL;
    if (rc) return rc;
    for (size_t i = 0; i < n; i++) load_row(e->C, rows[i]);
    return RA_OK;
}

extern "C" int ra_engine_read_rows(ra_engine* e, ra_row_state* rows, size_t n)
{
    if (!e || !rows_ok(e->C, rows, n)) return RA_E_INVAL;
    for (size_t i = 0; i < n; i++) read_row(e->C, rows[i]);
    return RA_OK;
}

extern "C" int ra_engine_load_query_state(ra_engine* e, const ra_query_state* q, size_t n)
{
    if (!e || !rows_ok(e->C, q, n)) return RA_E_INVAL;
    for (size_t i = 0; i < n; i++) load_query_row(e->C, q[i]);
    return RA_OK;
}

extern "C" int ra_engine_read_query_state(ra_engine* e, ra_query_state* q, size_t n)
{
    if (!e || !rows_ok(e->C, q, n)) return RA_E_INVAL;
    for (size_t i = 0; i < n; i++) read_query_row(e->C, q[i]);
    return RA_OK;
}

// ---- one row through one step: raft_step_kernel, then raft_general_kernel if it stalled -------

struct Scratch { ulonglong2 nm[RA_MAX_MEMBERS]; u64 cs[RA_MAX_MEMBERS]; };   // the per-thread shared-memory columns

// test observability: rows stepped by the narrow pass, records it refused (a field >= 2^30), rows it left to the
// general kernel because their sticky `wide` byte is set
static unsigned long long g_narrow_stats[3];
extern "C" void ra_emu_narrow_stats(unsigned long long* out, int reset)
{ for (int i = 0; i < 3; i++) { out[i] = g_narrow_stats[i]; if (reset) g_narrow_stats[i] = 0; } }
// test observability: stall contexts handed to the general kernel, and those of them whose wk_hi (the per-peer "sent a
// record that is not short" bits) is not zero
static unsigned long long g_stall_stats[2];
extern "C" void ra_emu_stall_stats(unsigned long long* out, int reset)
{ for (int i = 0; i < 2; i++) { out[i] = g_stall_stats[i]; if (reset) g_stall_stats[i] = 0; } }

// The hot kernel's fetch (raft_step_kernel.cuh): per record tile and plane, TMA stages 512 B (chunk 0), 1 KB (chunks
// 0-1) or 2 KB (chunks 0-3), as the size flags the warp ORs over its tile say.  The rest of the staging slot holds an
// earlier tile's bytes.  step_row reads a poison pattern there instead of the record, so a size flag that a writer
// failed to set shows as a result that differs from the oracle.  The poison decodes to values below 2^30: the narrow
// pass must take it for a plausible record rather than refuse it to the general path (which reads the plane again).
// (Which planes a tile fetches, and the ring's depth, do not matter: a row reads only its own planes, and every byte
// past the fetched length is poison whatever the slot held before.)
// Whether a poisoned record changes the outcome depends on the record; the count of records the hot path decoded
// from bytes the kernel would not have fetched does not (ra_emu_fetch_stats: it stays 0 while every flag is right).
static int g_poison;
static unsigned long long g_underfetch;
extern "C" void ra_emu_set_fetch_poison(int pattern) { g_poison = pattern; }
extern "C" void ra_emu_fetch_stats(unsigned long long* out, int reset) { out[0] = g_underfetch; if (reset) g_underfetch = 0; }
static ulonglong2 fetch_poison(u32 chunk, u32 row)
{
    if (g_poison == 0) return make_ulonglong2(2 * chunk + 1, 2 * chunk + 2);
    return make_ulonglong2(0x2345678u + 977u * row + chunk, 0x1234567u + 131u * row + 7u * chunk);
}
// the warp's size flags (raft_step_kernel.cuh: w_tail): bit s / 16 + s: a record from sender slot s has a tail / is
// not short; bit 8 + k / 24 + k: the same for host slot k.  Taken at the start of the tile, before any of its rows runs.
static u32 tile_sizes(const Cols& C, int cur, u32 r0)
{
    u32 w = 0;
    for (u32 r = r0; r < r0 + RT && r < C.rows; r++) {
        if (MT_FATAL(C.ap[r].y)) continue;
        const u64 cntw = C.routed ? C.mbox_cnt[cur][r] : 0;
        const u32 nloc = C.loc_n[r];
        for (u32 s = 0; s < C.members; s++) {
            const u32 c = (u32)(cntw >> (8 * s)) & 0xffu;
            w |= (((c >> 3) & 1u) | (((c >> 4) & 1u) << 16)) << s;
        }
        w |= (nloc & 0x0f00u) | ((nloc & 0xf000u) << 12);
    }
    return w;
}

namespace ra_wide {
#define RA_NARROW_PASS 0
#include "step_row.inc"
#undef RA_NARROW_PASS
}
namespace ra_narrow {
#define RA_NARROW_PASS 1
#include "step_row.inc"
#undef RA_NARROW_PASS
}
// a value left or entered the 32-bit pass out of range: the guards (Cols::wf, rec_decode) have a hole
extern "C" void ra_emu_narrow_violation(const char* what, unsigned long long v)
{
    fprintf(stderr, "ra_emu: narrow pass violation in %s(): value %llu\n", what, v);
    abort();
}

// the general kernel's body for one stall context (engine.cu: raft_general_kernel)
static void general_row(const Cols& C, int cur, const FloodArgs& F, const StallCtx& ctx)
{
    constexpr int MM = MK_MM(0, TR_RUNTIME);
    Scratch sc;
    const u32 r = ctx.row, flags = ctx.flags;
    u32 rem_mbox = ctx.rem_mbox, rem_loc = ctx.rem_loc;
    Member m;
    member_init(m, C, r, C.tc[r], C.lg[r], C.lw[r], C.ap[r], 0, cur, sc.nm);
    m.lrs_ok = 0;
    m.n_msgs = ctx.n_msgs_notes & 0xffffu; m.n_notes = (ctx.n_msgs_notes >> 16) & 0xffffu; m.status = ctx.status;
    m.sent_to = ctx.sent_to;
    { const u32 w = ctx.pn_type_slot_wk; m.pn_type = w & 0xffu; m.pn_slot = (w >> 8) & 0xffu; m.wk = (w >> 16) | ((u32)ctx.wk_hi << 16); }
    m.pn_a = ctx.pn_a; m.pn_b = ctx.pn_b; m.pn_c = ctx.pn_c;
    u64 big = 0;
    if (flags & STALL_PENDING) {
        MT_SET(m.meta, 24, 1, 0);
        process_event<MM>(m, mk_rec(r, RA_EV_PIPELINE_RPCS, RA_NO_SLOT, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0));
        m.cold &= ~8u;
    }
    while (rem_mbox) {
        const u32 p = __ffs(rem_mbox) - 1; rem_mbox &= rem_mbox - 1;
        const Rec e = ld_rec_plane(C.mbox[cur], C.tiles, p, r);
        big |= rec_magnitude(e);
        if (MT_FATAL(m.meta)) m.c_pack += 1u;
        else if (flood_lost<MM>(F, C, m, r, e)) m.c_pack += 1u << 20;
        else if (!note_budget_ok(m)) budget_drop_record(m);
        else if (C.pure || !fast_event<MM>(m, e)) { process_event<MM>(m, e); m.cold &= ~8u; }
    }
    while (rem_loc) {
        const u32 p = __ffs(rem_loc) - 1; rem_loc &= rem_loc - 1;
        const Rec e = ld_rec_plane(C.loc, C.tiles, p, r);
        big |= rec_magnitude(e);
        if (MT_FATAL(m.meta)) m.c_pack += 1u;
        else if (!note_budget_ok(m)) budget_refuse_local(m);
        else if (C.pure || !fast_event<MM>(m, e)) { process_event<MM>(m, e); m.cold &= ~8u; }
    }
    peers_writeback<MM>(m);
    const u32 k_fatal = row_end_of_step<MM>(m, C, r, cur, F);
    member_writeback(m, C, r);
    row_mark_wide(C, r, m, big);
    ra_wide::add_counters(C, m, k_fatal);
}

static int run_step(ra_engine* e, const FloodArgs& F)
{
    const Cols& C = e->C;
    if (C.n_shards > 1 && !C.peer_mode) {
        if (!C.outbox) return RA_E_INVAL;                       // ra_engine_set_outbox / ra_engine_peer_set first
        memset(C.out_cnt, 0, C.n_shards * sizeof(u32));
    }
    // M = 5 picks its specialisation by transport as the table k_step_kernels in engine.cu does; other M run runtime-M
    const int tr = step_transport(C);
    u32 w_tail = 0;
    for (u32 r = 0; r < C.rows; r++) {
        if ((r & (RT - 1)) == 0) w_tail = tile_sizes(C, e->cur, r);
        StallCtx ctx;
        bool stalled;
        if (C.members == 5) {
            switch (tr) {
            // (narrow pass for the same specialisations as launch_step(); RA_STEP_WIDE=1 keeps the 64-bit pass)
            case TR_LOCAL:  stalled = e->narrow ? ra_narrow::step_row<MK_MM(5, TR_LOCAL)>(C, e->cur, F, r, w_tail, ctx)
                                                : ra_wide::step_row<MK_MM(5, TR_LOCAL)>(C, e->cur, F, r, w_tail, ctx); break;
            case TR_PEER:   stalled = e->narrow ? ra_narrow::step_row<MK_MM(5, TR_PEER)>(C, e->cur, F, r, w_tail, ctx)
                                                : ra_wide::step_row<MK_MM(5, TR_PEER)>(C, e->cur, F, r, w_tail, ctx); break;
            case TR_BUCKET: stalled = ra_wide::step_row<MK_MM(5, TR_BUCKET)>(C, e->cur, F, r, w_tail, ctx); break;
            default:        stalled = e->narrow ? ra_narrow::step_row<MK_MM(5, TR_HOST)>(C, e->cur, F, r, w_tail, ctx)
                                                : ra_wide::step_row<MK_MM(5, TR_HOST)>(C, e->cur, F, r, w_tail, ctx); break;
            }
        } else stalled = ra_wide::step_row<MK_MM(0, TR_RUNTIME)>(C, e->cur, F, r, w_tail, ctx);
        // the general kernel runs after the step kernel; rows only ever write to OTHER rows' mailboxes of
        // the NEXT step, so handling a stalled row right away is the same thing
        if (stalled) general_row(C, e->cur, F, ctx);
    }
    if (C.routed) e->cur ^= 1;
    e->steps++;
    return RA_OK;
}

extern "C" int ra_engine_set_outbox(ra_engine* e, void* outbox, uint32_t* counts, uint32_t cap)
{ return e ? cols_set_outbox(e->C, outbox, counts, cap) : RA_E_INVAL; }

extern "C" int ra_engine_deliver(ra_engine* e, const void* inbox, const uint32_t* counts, uint32_t cap)
{
    if (!e || !deliver_args_ok(e->C, inbox, counts, cap)) return RA_E_INVAL;
    const ra_event* in = (const ra_event*)inbox;
    // e->cur is the buffer the next step reads: the one the last step's senders wrote into
    for (u32 b = 0; b < e->C.n_shards; b++) {
        const u32 n = counts[b] < cap ? counts[b] : cap;
        for (u32 i = 0; i < n; i++) deliver_record(e->C, e->cur, ld_rec(&in[(size_t)b * cap + i]));
    }
    return RA_OK;
}

// the peer transport (engine.cu: ra_engine_peer_get / ra_engine_peer_set): host pointers in place of device ones
extern "C" int ra_engine_peer_get(ra_engine* e, ra_peer_ptrs* out)
{ return e ? cols_peer_get(e->C, out) : RA_E_INVAL; }

extern "C" int ra_engine_peer_set(ra_engine* e, uint32_t shard, const ra_peer_ptrs* p)
{ return e ? cols_peer_set(e->C, shard, p) : RA_E_INVAL; }

// scan + gather_out: per-row slots -> flat arrays ordered by (row, seq).  When they do not fit, nothing is
// written and the slots stay: RA_E_CAPACITY with the sizes needed, the caller fetches again (engine.cu)
static int gather_out(ra_engine* e, ra_event* msgs, size_t msgs_cap, size_t* n_msgs,
                      ra_note* notes, size_t notes_cap, size_t* n_notes)
{
    const Cols& C = e->C;
    const u32 R = C.rows;
    size_t tm = 0, tn = 0;
    for (u32 r = 0; r < R; r++) { tm += C.out_n[r] & 0xffffu; tn += C.out_n[r] >> 16; }
    if (n_msgs) *n_msgs = tm;
    if (n_notes) *n_notes = tn;
    if (tm > msgs_cap || tn > notes_cap) { e->out_pending = 1; return RA_E_CAPACITY; }
    e->out_pending = 0;
    size_t om = 0, on = 0;
    for (u32 r = 0; r < R; r++) {
        const u32 v = C.out_n[r];
        C.out_n[r] = 0;
        const u32 nm = v & 0xffffu, nn = v >> 16;
        for (u32 k = 0; k < nm; k++) st_rec(&msgs[om + k], ld_rec(&C.omsg[(size_t)k * C.rows + r]));
        for (u32 k = 0; k < nn; k++) notes[on + k] = C.onote[(size_t)k * C.rows + r];
        om += nm; on += nn;
    }
    return RA_OK;
}

// ra_engine_fetch_output: nothing pending = nothing to fetch; RA_E_BUSY while calls submitted behind the one whose
// outputs did not fit are still to be collected
extern "C" int ra_engine_fetch_output(ra_engine* e, ra_event* msgs, size_t msgs_cap, size_t* n_msgs,
                                      ra_note* notes, size_t notes_cap, size_t* n_notes)
{
    if (!e || (!msgs && msgs_cap) || (!notes && notes_cap)) return RA_E_INVAL;
    if (!e->out_pending) { if (n_msgs) *n_msgs = 0; if (n_notes) *n_notes = 0; return RA_OK; }
    if (e->sub_n) return RA_E_BUSY;
    return gather_out(e, msgs, msgs_cap, n_msgs, notes, notes_cap, n_notes);
}

// ra_engine_pending_output: the sizes of outputs a call left in the slots (RA_E_CAPACITY), 0 / 0 otherwise
extern "C" int ra_engine_pending_output(ra_engine* e, size_t* n_msgs, size_t* n_notes)
{
    if (!e) return RA_E_INVAL;
    size_t tm = 0, tn = 0;
    for (u32 r = 0; e->out_pending && r < e->C.rows; r++) { tm += e->C.out_n[r] & 0xffffu; tn += e->C.out_n[r] >> 16; }
    if (n_msgs) *n_msgs = tm;
    if (n_notes) *n_notes = tn;
    return RA_OK;
}

// one call: ingest, the step, the gather (what submit_impl enqueues), for either record form (ra_event, ra_host_event)
template <typename EV>
static int eval_step(ra_engine* e, const EV* ev, size_t n_ev,
                     ra_event* msgs, size_t msgs_cap, size_t* n_msgs,
                     ra_note* notes, size_t notes_cap, size_t* n_notes)
{
    if ((!ev && n_ev) || n_ev > 0x7fffffffull) return RA_E_INVAL;
    const Cols& C = e->C;
    const u32 R = C.rows;
    // clear_loc_kernel, and (after a flood, whose last step wrote every row's out_n) the out_n clear of submit_impl
    for (u32 r = 0; r < R; r++) { C.loc_n[r] = 0; C.out_n[r] = 0; }
    u32 err = 0;
    for (u32 i = 0; i < (u32)n_ev; i++) ingest_event(C, ev, (u32)n_ev, i, &err);   // ingest_kernel, one event at a time
    if (err) {
        for (u32 r = 0; r < R; r++) C.loc_n[r] = 0;
        return err == 1 ? RA_E_UNGROUPED : (err == 2 ? RA_E_CAPACITY : RA_E_INVAL);
    }
    FloodArgs F; memset(&F, 0, sizeof F);
    { const int rc = run_step(e, F); if (rc) return rc; }
    return gather_out(e, msgs, msgs_cap, n_msgs, notes, notes_cap, n_notes);
}

// step = submit + collect (engine.cu: step_impl): not while a submitted call waits to be collected, nor while the
// outputs of an earlier call wait to be fetched
template <typename EV>
static int step_impl(ra_engine* e, const EV* ev, size_t n_ev, ra_event* msgs, size_t msgs_cap, size_t* n_msgs,
                     ra_note* notes, size_t notes_cap, size_t* n_notes)
{
    if (!e) return RA_E_INVAL;
    if (e->sub_n) return RA_E_BUSY;
    if (e->out_pending) return RA_E_CAPACITY;                    // ra_engine_fetch_output first
    return eval_step(e, ev, n_ev, msgs, msgs_cap, n_msgs, notes, notes_cap, n_notes);
}
extern "C" int ra_engine_step(ra_engine* e, const ra_event* ev, size_t n_ev, ra_event* msgs, size_t msgs_cap,
                              size_t* n_msgs, ra_note* notes, size_t notes_cap, size_t* n_notes)
{ return step_impl(e, ev, n_ev, msgs, msgs_cap, n_msgs, notes, notes_cap, n_notes); }
extern "C" int ra_engine_step_host(ra_engine* e, const ra_host_event* ev, size_t n_ev, ra_event* msgs, size_t msgs_cap,
                                   size_t* n_msgs, ra_note* notes, size_t notes_cap, size_t* n_notes)
{ return step_impl(e, ev, n_ev, msgs, msgs_cap, n_msgs, notes, notes_cap, n_notes); }

extern "C" int ra_engine_flood(ra_engine* e, uint32_t n_steps, uint32_t cmds_per_step, uint32_t election_permille,
                               uint64_t seed)
{ return ra_engine_flood_faults(e, n_steps, cmds_per_step, election_permille, seed, nullptr); }
extern "C" int ra_engine_flood_faults(ra_engine* e, uint32_t n_steps, uint32_t cmds_per_step, uint32_t election_permille,
                                      uint64_t seed, const ra_flood_faults* ff)
{
    FloodArgs F;
    const int rc0 = e ? flood_args(e->C, ff, cmds_per_step, election_permille, seed, F) : RA_E_INVAL;
    if (rc0) return rc0;
    for (u32 t = 0; t < n_steps; t++) {
        F.step = e->step_no + t;
        const int rc = run_step(e, F);
        if (rc) return rc;
    }
    e->step_no += n_steps;
    return RA_OK;
}

extern "C" int ra_engine_counters(ra_engine* e, ra_counters* out)
{
    if (!e || !out) return RA_E_INVAL;
    counters_unpack(e->C.counters, e->steps, out);
    return RA_OK;
}

extern "C" int ra_engine_stall_histogram(ra_engine* e, uint64_t* out128)
{
    if (!e || !out128) return RA_E_INVAL;
    memcpy(out128, e->C.counters + RA_CNT_STALL, (RA_CNT_REF - RA_CNT_STALL) * sizeof(u64));
    return RA_OK;
}

/* ---- the record-plane codec on its own: one ABI record through st_rec_plane / ld_rec_plane ---------- */
extern "C" int ra_emu_codec_roundtrip(const ra_event* in, ra_event* out, int* had_tail)
{
    if (!in || !out) return RA_E_INVAL;
    static thread_local ulonglong2 plane[4 * RT];              // one tile of one plane
    memset(plane, 0xA5, sizeof plane);                         // stale bytes must not leak into the result
    const u32 row = in->row & (RT - 1);
    const bool tail = st_rec_plane(plane, 1, 0, row, ld_rec(in));
    if (had_tail) *had_tail = tail ? 1 : 0;
    st_rec(out, ld_rec_plane(plane, 1, 0, row));
    return RA_OK;
}
/* the split-phase calls with the two-slot contract of include/ra_engine.h: the emulation evaluates a call when it is
 * submitted and hands the result over at collect.  A call submitted behind a rejected one gets the same status, one
 * submitted behind a call whose outputs did not fit gets RA_E_PENDING; neither is evaluated. */
template <typename EV>
static int submit_call(ra_engine* m, const EV* ev, size_t n_ev, ra_event* msgs, size_t msgs_cap, ra_note* notes, size_t notes_cap)
{
    if (!m || (!msgs && msgs_cap) || (!notes && notes_cap)) return RA_E_INVAL;
    if (m->out_pending && !m->out_held) return RA_E_CAPACITY;   // ra_engine_fetch_output first
    if (m->sub_n >= 2) return RA_E_BUSY;
    auto& s = m->sub[m->sub_n++];
    s.nm = s.nn = 0;
    if (m->sub_abort) { s.rc = m->sub_abort; return RA_OK; }
    s.rc = eval_step(m, ev, n_ev, msgs, msgs_cap, &s.nm, notes, notes_cap, &s.nn);
    if (s.rc == RA_E_CAPACITY && m->out_pending) { m->sub_abort = RA_E_PENDING; m->out_held = 1; }
    else if (s.rc) m->sub_abort = s.rc;
    return RA_OK;
}
extern "C" int ra_engine_submit_host(ra_engine* e, const ra_host_event* ev, size_t n_ev, ra_event* msgs, size_t msgs_cap,
                                     ra_note* notes, size_t notes_cap)
{ return submit_call(e, ev, n_ev, msgs, msgs_cap, notes, notes_cap); }
extern "C" int ra_engine_submit(ra_engine* e, const ra_event* ev, size_t n_ev, ra_event* msgs, size_t msgs_cap,
                                ra_note* notes, size_t notes_cap)
{ return submit_call(e, ev, n_ev, msgs, msgs_cap, notes, notes_cap); }
extern "C" int ra_engine_submit_host_segs(ra_engine* e, const ra_host_event_seg* segs, size_t n_segs, ra_event* msgs,
                                          size_t msgs_cap, ra_note* notes, size_t notes_cap)
{
    if (!host_segs_ok(segs, n_segs)) return RA_E_INVAL;
    size_t n = 0;
    for (size_t k = 0; k < n_segs; k++) n += segs[k].n;
    ra_host_event* all = (ra_host_event*)malloc((n ? n : 1) * sizeof(ra_host_event));
    if (!all) return RA_E_NOMEM;
    size_t off = 0;
    for (size_t k = 0; k < n_segs; k++) { if (segs[k].n) memcpy(all + off, segs[k].ev, segs[k].n * sizeof(ra_host_event)); off += segs[k].n; }
    const int rc = ra_engine_submit_host(e, all, n, msgs, msgs_cap, notes, notes_cap);
    free(all);
    return rc;
}
extern "C" int ra_engine_collect(ra_engine* e, size_t* n_msgs, size_t* n_notes)
{
    if (!e || !e->sub_n) return RA_E_INVAL;                      // nothing submitted
    const auto s = e->sub[0];
    e->sub[0] = e->sub[1];
    if (--e->sub_n == 0) e->sub_abort = 0;
    if (s.rc == RA_E_CAPACITY && e->out_held) e->out_held = 0;   // the caller learns of the outputs waiting to be fetched
    if (n_msgs) *n_msgs = s.nm;
    if (n_notes) *n_notes = s.nn;
    return s.rc;
}
