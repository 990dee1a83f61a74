/*
 * ra_oracle.c -- TEST INFRASTRUCTURE ONLY (see ra_oracle.h).
 *
 * Plain-C restatement of the reference's Raft decision logic
 *   rabbitmq/ra v3.1.6  src/ra_server.erl  (handle_leader/2, handle_follower/2,
 *   handle_candidate/2, handle_pre_vote/2, handle_await_condition/2 and helpers)
 * over a literal index->term map log model that follows the ra_log facade
 *   src/ra_log.erl (fetch_term :1140-1152, exists :1413-1419, write :543-566,
 *   set_last_index :800-845, handle_event{written} :849-896, next_index :1119)
 * and the suite's fake, test/ra_log_memory.erl:74-233.
 *
 * Every function cites the clause it restates.  The structure deliberately
 * mirrors the Erlang (one C function per Erlang function, one branch per
 * clause, AoS member structs, a per-index term array) and shares NO code with
 * ra_b200/csrc: the CUDA engine keeps SoA columns and a run-length log view.
 *
 * Parity pinning: tests/test_golden_*.py replay the reference's own vectors
 * (test/ra_server_SUITE.erl, src/ra_server.erl:4198-4211) against this file.
 *
 * Where ra_log_memory and the production ra_log disagree, production wins:
 *   - fetch_term/2 answers only inside the log range (ra_log.erl:1140-1152);
 *     ra_log_memory keeps stale map entries above last_index after
 *     set_last_index/2.
 *   - set_last_index/2 re-reads the term of min(Idx, LastWrittenIdx)
 *     (ra_log.erl:827-845); ra_log_memory only rewinds when Idx < LWIdx.
 *   - a written event whose last index is at or below the snapshot index and
 *     no longer in the log is a no-op (ra_log.erl:871-881).
 * Out of scope (host side, flagged not guessed): ra_log's `pending` ARQ
 * sequence (:860-869), payloads, cluster-change entries, machine versions > 0,
 * snapshot installation, consistent queries.
 *
 * Engine-contract items that are not in the reference and are implemented by
 * both backends from the text of DESIGN.md ("contract" section):
 *   - an AER record spans at most two term runs (batch cut at the 2nd boundary);
 *   - the log view keeps at most RA_MAX_RUNS term runs (oldest forgotten);
 *   - at most one chased pipeline_rpcs pass per input event, remainder deferred;
 *   - transport capacities RA_MSG_CAP / RA_MBOX_DEPTH (drop + count when full).
 */
#define _GNU_SOURCE
#include "ra_oracle.h"
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

typedef uint64_t u64;
typedef int64_t  i64;
typedef uint32_t u32;
typedef uint8_t  u8;

#define UNDEF RA_UNDEF_TERM

/* ------------------------------------------------------------------ */
/* member state: ra_server_state() src/ra_server.erl:73-112            */
/* ------------------------------------------------------------------ */
typedef struct {
    u64 next_index, match_index, commit_index_sent;
    u64 query_index;                 /* consistent queries, ra.hrl:63-75 */
    u8  status, voter;
} peer_t;

typedef struct {
    /* the log facade: literal per-index terms for [first_index,last_index] */
    u64 *terms;          /* terms[i - store_base] */
    u64  store_base;
    size_t store_cap;
    u64 first_index, last_index, last_term;
    u64 lw_idx, lw_term;             /* last_written_index_term */
    u8  has_snapshot;
    u64 snap_idx, snap_term;         /* ra_snapshot:current/1 */
    u32 n_runs;                      /* contract: horizon of RA_MAX_RUNS runs */
} log_t;

typedef struct {
    u32 row;
    u8  role, self_slot, n_members, leader_slot, voted_for, membership;
    u8  condition;                   /* follower_catchup_cond_fun(Reason) :2179 */
    u8  cond_reply_valid;
    u8  pipeline_pending;
    u8  fatal;
    u32 votes, machine_version, effective_machine_version;
    u64 current_term, commit_index, last_applied;
    u64 pre_vote_token, token_counter;
    u64 query_index;                 /* ra_server_state() :96 */
    u64 agreed_index;                /* highest query index a quorum confirmed and the host was told */
    u64 cond_reply_term, cond_reply_next, cond_reply_last_index, cond_reply_last_term;
    peer_t peers[RA_MAX_MEMBERS];
    log_t log;
    u32 idle;                        /* flood host model: election timer */
} member_t;

struct ra_oracle {
    ra_engine_cfg cfg;
    u32 n_rows;
    member_t *m;
    ra_counters cnt;
    /* routed transport: mailbox[buf][(src*DEPTH+k)*n_rows + row] */
    ra_event *mbox[2];
    u8 *mbox_n[2];                   /* [src*n_rows + row] */
    int cur;                         /* buffer read this step */
    /* flood host model: locals for the next flood step */
    ra_event *loc;                   /* [k*n_rows + row] */
    u8 *loc_n;
    u64 step_no;
    u32 note_cap;                    /* notes per row per step (cfg.note_cap or RA_NOTE_CAP) */
    /* sample view (ra_oracle_set_sample): local group g stands for global group offset + g * stride of a run
       over total_groups groups; the flood host model is keyed by the GLOBAL group / row ids */
    u32 s_stride, s_offset, s_total;
};

/* flood fault injection (include/ra_engine.h, ra_flood_faults): contract, keyed by global ids */
struct flood_faults { u32 drop, withhold, part, part_len; };

/* per-row, per-step output context */
typedef struct {
    ra_oracle *o;
    member_t *m;
    ra_event msgs[RA_MSG_CAP];  u32 n_msgs;
    ra_note  notes[RA_NOTE_CAP]; u32 n_notes;
    u32 status;                 /* RA_ST_* */
    u32 fatal_code;
    u32 unconsumed;             /* host events refused by the note budget */
    const struct flood_faults *ff; /* fault injection of the flood in progress (NULL otherwise) */
    u64 ff_seed, ff_step;
    u8  role_at_start;
    u8  sent_to[RA_MAX_MEMBERS]; /* routed mode: records put in (self -> slot) mailbox */
    ra_counters *cnt;
    int routed_out;              /* deliver through mailboxes */
} ctx_t;

/* a raft message as handled by ra_server: reuse the wire record */
typedef ra_event msg_t;

/* ------------------------------------------------------------------ */
/* log facade                                                          */
/* ------------------------------------------------------------------ */
static void log_reserve(log_t *l, u64 idx)
{
    if (l->store_cap == 0) {
        l->store_cap = 16;
        l->terms = (u64 *)malloc(l->store_cap * sizeof(u64));
        l->store_base = l->first_index;
    }
    /* drop storage below first_index when it is at least half of the store */
    if (l->first_index > l->store_base && l->first_index - l->store_base > l->store_cap / 2) {
        u64 shift = l->first_index - l->store_base;
        u64 live = (l->last_index + 1 > l->first_index) ? l->last_index + 1 - l->first_index : 0;
        if (live) memmove(l->terms, l->terms + shift, live * sizeof(u64));
        l->store_base = l->first_index;
    }
    while (idx - l->store_base >= l->store_cap) {
        l->store_cap *= 2;
        l->terms = (u64 *)realloc(l->terms, l->store_cap * sizeof(u64));
    }
}

static int log_in_range(const log_t *l, u64 idx)
{   /* ?IS_IN_RANGE ra_log.erl:470-473 */
    return l->first_index <= l->last_index && idx >= l->first_index && idx <= l->last_index;
}

/* ra_log:fetch_term/2  ra_log.erl:1140-1152 */
static u64 log_fetch_term(const log_t *l, i64 idx)
{
    if (idx < 0) return UNDEF;
    if (!log_in_range(l, (u64)idx)) return UNDEF;
    return l->terms[(u64)idx - l->store_base];
}

/* ra_log:exists/2  ra_log.erl:1413-1419 */
static int log_exists(const log_t *l, u64 idx, u64 term)
{
    u64 t = log_fetch_term(l, (i64)idx);
    return t != UNDEF && t == term;
}

/* ra_log:next_index/1  ra_log.erl:1118-1126 */
static u64 log_next_index(const log_t *l) { return l->last_index + 1; }

/* contract: forget the oldest term run when more than RA_MAX_RUNS are held */
static void log_enforce_horizon(log_t *l)
{
    while (l->n_runs > RA_MAX_RUNS) {
        u64 i = l->first_index;
        u64 t = l->terms[i - l->store_base];
        while (i <= l->last_index && l->terms[i - l->store_base] == t) i++;
        l->first_index = i;
        l->n_runs--;
    }
}

/* append one entry at last_index+1 (tail of ra_log:append/2 and of write/2) */
static void log_push(log_t *l, u64 idx, u64 term)
{
    int empty = !(l->first_index <= l->last_index);
    if (empty) { l->first_index = idx; l->store_base = idx; }   /* nothing live: restart the window */
    log_reserve(l, idx);
    l->terms[idx - l->store_base] = term;
    if (empty || term != l->last_term || l->n_runs == 0) l->n_runs++;
    l->last_index = idx;
    l->last_term = term;
    log_enforce_horizon(l);
}

/* drop everything above idx (range limit, ra_range:limit(Idx+1, Range)) */
static void log_truncate(log_t *l, u64 idx, u64 term_at_idx)
{
    for (u64 i = l->last_index; i > idx && i >= l->first_index; i--) {
        if (i == l->first_index || l->terms[i - 1 - l->store_base] != l->terms[i - l->store_base])
            l->n_runs--;
        if (i == 0) break;
    }
    l->last_index = idx;
    l->last_term = term_at_idx;
    if (idx < l->first_index) {          /* log now empty: range undefined */
        l->first_index = idx + 1;
        l->n_runs = 0;
    }
}

/* ra_log:snapshot_index_term/1 */
static int log_snapshot(const log_t *l, u64 *idx, u64 *term)
{
    if (!l->has_snapshot) return 0;
    *idx = l->snap_idx; *term = l->snap_term;
    return 1;
}

/* ra_log:set_last_index/2  ra_log.erl:800-845.  returns 0 = {not_found,_} */
static int log_set_last_index(log_t *l, u64 idx)
{
    u64 t = log_fetch_term(l, (i64)idx);
    u64 si, st;
    int has = log_snapshot(l, &si, &st);
    if (t == UNDEF && !(has && si == idx)) return 0;            /* :816-818 */
    if (has && si == idx) {                                     /* :819-829 */
        log_truncate(l, idx, st);
        l->lw_idx = si; l->lw_term = st;
        return 1;
    }
    /* :830-845 */
    u64 lwidx = idx < l->lw_idx ? idx : l->lw_idx;
    u64 lwterm;
    if (has && si == lwidx) lwterm = st;
    else lwterm = log_fetch_term(l, (i64)lwidx);
    log_truncate(l, idx, t);
    l->lw_idx = lwidx; l->lw_term = lwterm;                     /* true = LWTerm =/= undefined */
    return 1;
}

/* ra_log:handle_event({written,Term,[{From,To}]})  ra_log.erl:849-896,
   test/ra_log_memory.erl:196-209 */
static void log_handle_written(log_t *l, u64 term, u64 from, u64 to)
{
    u64 idx = to;                                               /* ra_seq:last/1 */
    for (;;) {
        u64 t = log_fetch_term(l, (i64)idx);
        if (t != UNDEF && t == term) {                          /* :861-870 */
            l->lw_idx = idx; l->lw_term = term;
            return;
        }
        if (t == UNDEF && l->has_snapshot && idx <= l->snap_idx) /* :871-881 */
            return;
        /* term mismatch: ra_seq:limit(Idx - 1, Seq)  :882-895 */
        if (idx == 0 || idx - 1 < from) return;
        idx = idx - 1;
    }
}

/* ------------------------------------------------------------------ */
/* small helpers of ra_server.erl                                      */
/* ------------------------------------------------------------------ */

/* ra_server:fetch_term/2 :3158-3169 (falls back on the snapshot) */
static u64 srv_fetch_term(const member_t *m, i64 idx)
{
    u64 t = log_fetch_term(&m->log, idx);
    if (t != UNDEF) return t;
    u64 si, st;
    if (idx >= 0 && log_snapshot(&m->log, &si, &st) && si == (u64)idx) return st;
    return UNDEF;
}

/* last_idx_term/1 :3039 -> ra_log:last_index_term/1 ra_log.erl:786-791 */
static void last_idx_term(const member_t *m, u64 *idx, u64 *term)
{
    *idx = m->log.last_index; *term = m->log.last_term;
}

/* agreed_commit/1 :3657-3661 */
uint64_t ra_oracle_agreed_commit(const uint64_t *indexes, size_t n)
{
    u64 s[RA_MAX_MEMBERS + 1];
    if (n == 0 || n > RA_MAX_MEMBERS + 1) return 0;
    memcpy(s, indexes, n * sizeof(u64));
    for (size_t i = 1; i < n; i++) {            /* lists:sort(fun erlang:'>'/2, _) */
        u64 v = s[i]; size_t j = i;
        while (j > 0 && s[j - 1] < v) { s[j] = s[j - 1]; j--; }
        s[j] = v;
    }
    size_t nth = n / 2 + 1;                      /* trunc(length/2) + 1 */
    return s[nth - 1];
}

/* count_voters/1 :3974-3982, required_quorum/1 :3969-3972 */
static u32 required_quorum(const member_t *m)
{
    u32 voters = 0;
    for (u32 s = 0; s < m->n_members; s++) if (m->peers[s].voter) voters++;
    return voters / 2 + 1;
}

static int is_peer(const member_t *m, u32 slot)
{   /* peer(PeerId, State) :3008 looks the id up in the cluster map (self included) */
    return slot < m->n_members;
}

/* ------------------------------------------------------------------ */
/* output helpers                                                      */
/* ------------------------------------------------------------------ */
static void set_fatal(ctx_t *c, u32 code)
{
    if (!(c->status & RA_ST_FATAL)) { c->status |= RA_ST_FATAL; c->fatal_code = code; }
    c->m->fatal = 1;
}

static void note(ctx_t *c, u8 type, u8 slot, u64 a, u64 b, u64 cc)
{
    /* contract: a WAL_APPEND that continues the previous note's range in the same term merges */
    if (type == RA_NOTE_WAL_APPEND && c->n_notes > 0) {
        ra_note *p = &c->notes[c->n_notes - 1];
        if (p->type == RA_NOTE_WAL_APPEND && p->c == cc && p->b + 1 == a) { p->b = b; return; }
    }
    if (type == RA_NOTE_APPLY && c->n_notes > 0) {
        ra_note *p = &c->notes[c->n_notes - 1];
        if (p->type == RA_NOTE_APPLY && p->b + 1 == a) { p->b = b; return; }
    }
    if (c->n_notes >= c->o->note_cap - 1) {
        /* contract (include/ra_engine.h, note budget): unreachable while an event stays within
           RA_NOTE_RESERVE notes; otherwise nothing is lost silently -- the row stops */
        c->status |= RA_ST_NOTE_OVERFLOW; set_fatal(c, RA_FATAL_NOTE_OVERFLOW); return;
    }
    ra_note *n = &c->notes[c->n_notes++];
    n->row = c->m->row; n->type = type; n->slot = slot; n->aux = 0;
    n->a = a; n->b = b; n->c = cc;
}

/* contract: the note budget.  A row takes the next event of its step only while RA_NOTE_RESERVE
   slots + the STATUS slot are free; mailbox records it does not reach are dropped and counted,
   host events are left unconsumed (STATUS.c bits 8..15) */
static int note_budget_ok(const ctx_t *c) { return c->n_notes + RA_NOTE_RESERVE + 1u <= c->o->note_cap; }
static void budget_drop_record(ctx_t *c)
{ c->status |= RA_ST_NOTE_OVERFLOW | RA_ST_MSG_DROPPED; c->cnt->msgs_dropped++; }
static void budget_refuse_local(ctx_t *c) { c->status |= RA_ST_NOTE_OVERFLOW; c->unconsumed++; }
static void process_event(ctx_t *c, const ra_event *in);
static u64 mix64(u64 x);
static void flood_ids(const ctx_t *c, u64 *gg, u64 *gr)
{
    const ra_oracle *o = c->o; const member_t *m = c->m;
    u32 G = o->cfg.n_groups, g = m->row % G;
    *gg = g; *gr = m->row;
    if (o->s_stride) { *gg = (u64)o->s_offset + (u64)g * o->s_stride; *gr = (u64)m->self_slot * o->s_total + *gg; }
}
/* contract: is this mailbox record lost before the row evaluates it? */
static int flood_lost(const ctx_t *c, const ra_event *e)
{
    const struct flood_faults *f = c->ff;
    if (!f || !(f->drop | f->part)) return 0;
    u64 gg, gr; flood_ids(c, &gg, &gr);
    if (f->part) {
        u64 w = c->ff_step / f->part_len;
        u32 h = (u32)(mix64(c->ff_seed ^ (w * 0xC2B2AE3D27D4EB4Full) ^ (gg * 0x165667B19E3779F9ull)) >> 32);
        if (h % 1000u < f->part) { u32 p = (h / 1000u) % c->m->n_members; if (p == c->m->self_slot || p == e->from_slot) return 1; }
    }
    if (f->drop && e->type == RA_EV_AER) {
        u32 h = (u32)(mix64(c->ff_seed ^ (c->ff_step * 0x9E3779B97F4A7C15ull) ^ (gr * 0xD6E8FEB86659FD93ull) ^ ((u64)(e->from_slot + 1) << 56)) >> 32);
        if (h % 1000u < f->drop) return 1;
    }
    return 0;
}
static void take_record(ctx_t *c, const ra_event *e)
{
    if (!c->m->fatal && flood_lost(c, e)) { c->cnt->msgs_dropped++; return; }
    if (!c->m->fatal && !note_budget_ok(c)) budget_drop_record(c); else process_event(c, e);
}
static void take_local(ctx_t *c, const ra_event *e)
{ if (!c->m->fatal && !note_budget_ok(c)) budget_refuse_local(c); else process_event(c, e); }

static u32 row_of(const ra_oracle *o, u32 group, u32 slot) { return slot * o->cfg.n_groups + group; }
static u32 group_of(const ra_oracle *o, u32 row) { return row % o->cfg.n_groups; }

/* send one RPC record to the member in `to_slot` of my group */
static void emit_msg(ctx_t *c, u32 to_slot, msg_t *e)
{
    ra_oracle *o = c->o;
    member_t *m = c->m;
    e->row = row_of(o, group_of(o, m->row), to_slot);
    if (c->routed_out && !(e->flags & RA_EVF_NEXT_EVENT) && to_slot >= m->n_members)
        return;                                          /* no mailbox for an unknown peer */
    if (!(e->flags & RA_EVF_NEXT_EVENT)) e->from_slot = m->self_slot;
    e->_pad = 0;
    if (c->routed_out && !(e->flags & RA_EVF_NEXT_EVENT)) {
        u32 k = c->sent_to[to_slot];
        if (k >= RA_MBOX_DEPTH) { c->status |= RA_ST_MSG_DROPPED; c->cnt->msgs_dropped++; return; }
        int nb = o->cur ^ 1;
        e->seq = k;
        o->mbox[nb][((size_t)m->self_slot * RA_MBOX_DEPTH + k) * o->n_rows + e->row] = *e;
        c->sent_to[to_slot] = (u8)(k + 1);
        c->cnt->msgs_out++;
        return;
    }
    if (c->n_msgs >= RA_MSG_CAP) { c->status |= RA_ST_MSG_DROPPED; c->cnt->msgs_dropped++; return; }
    e->seq = c->n_msgs;
    c->msgs[c->n_msgs++] = *e;
    c->cnt->msgs_out++;
}

/* ------------------------------------------------------------------ */
/* term / vote                                                         */
/* ------------------------------------------------------------------ */

/* update_term_and_voted_for/3 :3014-3031 */
static void update_term_and_voted_for(ctx_t *c, u64 term, u8 voted_for)
{
    member_t *m = c->m;
    if (term == m->current_term && voted_for == m->voted_for) return;
    m->current_term = term;
    m->voted_for = voted_for;
    c->status |= RA_ST_TERM_VOTE_CHANGED;      /* ra_log_meta:store_sync :3024-3025 */
    c->cnt->term_and_voted_for_updates++;      /* :3026 */
    for (u32 p = 0; p < RA_MAX_MEMBERS; p++) m->peers[p].query_index = 0;   /* reset_query_index/1 :3029 */
}

/* update_term/2 :3033-3037 */
static void update_term(ctx_t *c, u64 term)
{
    if (term > c->m->current_term) update_term_and_voted_for(c, term, RA_NO_SLOT);
}

/* is_candidate_log_up_to_date/3 :3132-3139 */
static int is_candidate_log_up_to_date(u64 idx, u64 term, u64 last_idx, u64 last_term)
{
    if (term > last_term) return 1;
    if (term == last_term && idx >= last_idx) return 1;
    return 0;
}

/* ------------------------------------------------------------------ */
/* replies                                                             */
/* ------------------------------------------------------------------ */

/* append_entries_reply/3 :3597-3604 */
static msg_t make_aer_reply(const member_t *m, u64 term, int success)
{
    msg_t r; memset(&r, 0, sizeof r);
    r.type = RA_EV_AER_REPLY;
    r.term = term;
    r.a = m->log.last_index + 1;     /* next_index */
    r.b = m->log.lw_idx;             /* last_index = last written */
    r.c = m->log.lw_term;
    r.d = success ? 1 : 0;
    return r;
}

/* cast_reply/3 :3683 */
static void cast_reply(ctx_t *c, u32 to_slot, msg_t r) { emit_msg(c, to_slot, &r); }

static void reply_vote_result(ctx_t *c, u32 to_slot, u8 type, u64 term, u64 token, int granted)
{
    msg_t r; memset(&r, 0, sizeof r);
    r.type = type; r.term = term; r.c = token; r.d = granted ? 1 : 0;
    emit_msg(c, to_slot, &r);
}

/* a {next_event, Msg} effect: queued for the proc shim (or returned in pure mode) */
typedef struct { msg_t q[6]; u32 n; } nextq_t;

static void next_event(nextq_t *nq, const msg_t *msg, int info)
{
    if (nq->n < 6) {
        nq->q[nq->n] = *msg;
        if (info) nq->q[nq->n].flags |= RA_EVF_INFO;
        nq->n++;
    }
}

/* ------------------------------------------------------------------ */
/* apply_to / evaluate_quorum                                          */
/* ------------------------------------------------------------------ */

/* apply_to/3 :3217-3255 restricted to '$usr' and same-version noop entries: every
   entry in From..To advances last_applied (apply_with/2 :3289-3308, :3388-3390);
   the host runs ra_machine:apply/3 for the range in the APPLY note.             */
static void apply_to(ctx_t *c, u64 apply_to_idx)
{
    member_t *m = c->m;
    if (!(apply_to_idx > m->last_applied)) return;                       /* guard :3230 */
    if (!(m->machine_version >= m->effective_machine_version)) return;
    u64 from = m->last_applied + 1;
    u64 to = m->log.last_index < apply_to_idx ? m->log.last_index : apply_to_idx;
    if (to < from) return;                                               /* empty fold */
    note(c, RA_NOTE_APPLY, 0, from, to, 0);
    c->cnt->applied += to - from + 1;
    m->last_applied = to;
}

/* match_indexes/1 :3644-3655 + agreed_commit/1 + increment_commit_index/1 :3621-3630
   + evaluate_quorum/2 :3606-3619 */
static void evaluate_quorum(ctx_t *c)
{
    member_t *m = c->m;
    u64 ci0 = m->commit_index;
    u64 idxs[RA_MAX_MEMBERS + 1]; size_t n = 0;
    idxs[n++] = m->log.lw_idx;                                           /* [LWIdx] */
    for (u32 s = 0; s < m->n_members; s++) {
        if (s == m->self_slot) continue;
        if (!m->peers[s].voter) continue;
        idxs[n++] = m->peers[s].match_index;
    }
    u64 potential = ra_oracle_agreed_commit(idxs, n);
    if (srv_fetch_term(m, (i64)potential) == m->current_term)            /* §5.4.2 gate */
        m->commit_index = potential;
    if (m->commit_index > ci0) {                                         /* :3611-3614 */
        note(c, RA_NOTE_COMMIT, 0, ci0, m->commit_index, 0);
        c->cnt->commits += m->commit_index - ci0;
    }
    apply_to(c, m->commit_index);
}

/* evaluate_commit_index_follower/2 :2229-2263 */
static void evaluate_commit_index_follower(ctx_t *c)
{
    member_t *m = c->m;
    if (m->leader_slot == RA_NO_SLOT) return;                            /* :2261 */
    u64 idx = m->log.last_index;
    u64 at = idx < m->commit_index ? idx : m->commit_index;
    apply_to(c, at);
}

/* ------------------------------------------------------------------ */
/* leader: RPC generation                                              */
/* ------------------------------------------------------------------ */

/* make_append_entries_rpc/6 :2401-2418.  Returns the new next index (To + 1). */
static u64 make_append_entries_rpc(ctx_t *c, u32 peer, i64 prev_idx, u64 prev_term, u64 num)
{
    member_t *m = c->m;
    u64 last = m->log.last_index;
    u64 from = (u64)(prev_idx + 1);
    u64 to = (u64)prev_idx + num; if (last < to) to = last;              /* min(LastIndex, PrevIdx + Num) */
    if (to >= from && to - from >= 0xFFFFu) to = from + 0xFFFEu;        /* contract: <= 65535 entries per record */
    msg_t r; memset(&r, 0, sizeof r);
    r.type = RA_EV_AER;
    r.term = m->current_term;
    r.a = (u64)prev_idx; r.b = prev_term; r.c = m->commit_index;
    if (to >= from && log_in_range(&m->log, from)) {
        /* entry terms: contract = at most two runs per record */
        u64 t1 = log_fetch_term(&m->log, (i64)from);
        u64 i = from;
        while (i <= to && log_fetch_term(&m->log, (i64)i) == t1) i++;
        r.d = t1;
        if (i <= to) {
            u64 t2 = log_fetch_term(&m->log, (i64)i);
            u64 j = i;
            while (j <= to && log_fetch_term(&m->log, (i64)j) == t2) j++;
            r.n1 = (uint16_t)(i - from); r.e = t2;
            to = j - 1;                                                  /* cut at the 2nd boundary */
        }
        r.n = (uint16_t)(to - from + 1);
    } else {
        to = from - 1;                                                   /* no entries */
        if (last < to) to = last;
        r.n = 0;
    }
    emit_msg(c, peer, &r);
    return to + 1;
}

/* make_rpc_effect/5 :2365-2399.  *snapshot = 1 when a snapshot must be sent. */
static u64 make_rpc_effect(ctx_t *c, u32 peer, u64 next, u64 max_batch, int *snapshot)
{
    member_t *m = c->m;
    i64 prev_idx = (i64)next - 1;
    *snapshot = 0;
    u64 pt = log_fetch_term(&m->log, prev_idx);
    if (pt != UNDEF) return make_append_entries_rpc(c, peer, prev_idx, pt, max_batch);
    u64 si, st;
    if (!log_snapshot(&m->log, &si, &st)) {       /* case clause on `undefined` :2378 */
        set_fatal(c, RA_FATAL_NO_SNAPSHOT);
        return next;
    }
    if (prev_idx >= 0 && si == (u64)prev_idx)
        return make_append_entries_rpc(c, peer, prev_idx, st, max_batch);
    if (!(prev_idx < (i64)si)) { set_fatal(c, RA_FATAL_ASSERT); return next; }   /* ?assert :2390 */
    *snapshot = 1;
    note(c, RA_NOTE_SEND_SNAPSHOT, (u8)peer, peer, si, 0);
    return si;
}

/* make_pipelined_rpc_effects/3 :2268-2329.  Returns More. */
static int make_pipelined_rpc_effects(ctx_t *c, int force, int pure)
{
    member_t *m = c->m;
    u64 next_log_idx = log_next_index(&m->log);
    i64 max_pipe = c->o->cfg.max_pipeline_count;
    i64 max_batch = c->o->cfg.max_aer_batch;
    int more = 0;
    for (u32 s = 0; s < m->n_members; s++) {                 /* maps:fold over the cluster */
        peer_t *p = &m->peers[s];
        if (s == m->self_slot) continue;
        if (p->status != RA_PEER_NORMAL) continue;
        if (!(p->next_index < next_log_idx || p->commit_index_sent < m->commit_index)) continue;
        i64 in_flight = (i64)p->next_index - (i64)p->match_index - 1;
        if (!(in_flight < max_pipe || force)) continue;
        i64 bs = max_pipe - in_flight; if (max_batch < bs) bs = max_batch; if (bs < 1) bs = 1;
        int snap = 0;
        u64 new_next = make_rpc_effect(c, s, p->next_index, (u64)bs, &snap);
        if (c->m->fatal) return 0;
        if (!(new_next >= p->next_index)) { set_fatal(c, RA_FATAL_ASSERT); return 0; }  /* ?assert :2316 */
        p->next_index = new_next;
        p->commit_index_sent = m->commit_index;
        if (snap && !pure) p->status = RA_PEER_SENDING_SNAPSHOT;   /* ra_server_proc.erl:1719-1721 */
        i64 new_in_flight = (i64)new_next - (i64)p->match_index - 1;
        if (new_next < next_log_idx && new_in_flight < max_pipe) more = 1;
    }
    return more;
}

/* ---- consistent queries: the heartbeat round, :3700-3825 ------------------------------ */
static void send_heartbeat_reply(ctx_t *c, u32 to, u64 term, u64 query_index)
{   /* heartbeat_reply/2 :3700-3702, cast to the rpc's leader_id */
    msg_t r; memset(&r, 0, sizeof r);
    r.type = RA_EV_HEARTBEAT_REPLY; r.term = term; r.a = query_index;
    emit_msg(c, to, &r);
}
/* heartbeat_rpc_effects/4 :3749-3771: normal peers whose query_index lags */
static void heartbeat_rpc_effects(ctx_t *c, u64 query_index)
{
    member_t *m = c->m;
    for (u32 s = 0; s < m->n_members; s++) {
        if (s == m->self_slot) continue;
        if (m->peers[s].status != RA_PEER_NORMAL) continue;
        if (!(m->peers[s].query_index < query_index)) continue;
        msg_t r; memset(&r, 0, sizeof r);
        r.type = RA_EV_HEARTBEAT_RPC; r.term = m->current_term; r.a = query_index;
        emit_msg(c, s, &r);
    }
}
/* get_current_query_quorum/1 :3796-3797 over query_indexes/1 :3632-3642 */
static u64 query_quorum(const member_t *m)
{
    u64 v[RA_MAX_MEMBERS]; size_t n = 0;
    v[n++] = m->query_index;
    for (u32 s = 0; s < m->n_members; s++)
        if (s != m->self_slot && m->peers[s].voter) v[n++] = m->peers[s].query_index;
    return ra_oracle_agreed_commit(v, n);
}
/* what the waiting queries learn: every one with an index <= agreed is applied by the host */
static void query_agreed(ctx_t *c, u64 agreed)
{
    member_t *m = c->m;
    if (agreed > m->agreed_index) {
        m->agreed_index = agreed;
        note(c, RA_NOTE_QUERY_AGREED, 0, agreed, 0, 0);
    }
}
/* update_heartbeat_rpc_effects/1 :3704-3720 (tick, enforce leadership) */
static void update_heartbeat_rpc_effects(ctx_t *c)
{
    member_t *m = c->m;
    if (m->n_members <= 1) query_agreed(c, m->query_index);       /* no peers: apply everything waiting */
    else heartbeat_rpc_effects(c, m->query_index);
}

/* make_rpcs_for/2 :2352-2360 over stale_peers/1 :2985-3003 (all=0) or every normal
   peer (make_all_rpcs/1 :2337-2350, all=1); batch size 1, peers are not updated */
static void make_rpcs(ctx_t *c, int all)
{
    member_t *m = c->m;
    if (all)                                   /* make_all_rpcs/1: CancelEffects ++ EffectsAER ++ EffectsHR */
        for (u32 s = 0; s < m->n_members; s++)
            if (s != m->self_slot && m->peers[s].status == RA_PEER_SNAPSHOT_BACKOFF)
                note(c, RA_NOTE_CANCEL_SNAPSHOT_RETRY, (u8)s, s, 0, 0);
    for (u32 s = 0; s < m->n_members; s++) {
        peer_t *p = &m->peers[s];
        if (s == m->self_slot) continue;
        if (p->status != RA_PEER_NORMAL && !(all && p->status == RA_PEER_SNAPSHOT_BACKOFF)) continue;
        if (!all) {
            int stale = ((i64)p->match_index < (i64)p->next_index - 1) ||
                        (p->commit_index_sent < m->commit_index);
            if (!stale) continue;
        }
        int snap = 0;
        (void)make_rpc_effect(c, s, p->next_index, 1, &snap);
        if (c->m->fatal) return;
    }
    update_heartbeat_rpc_effects(c);                          /* EffectsAER ++ EffectsHR */
}

/* initialise_peers/1 :3207-3215 */
static void initialise_peers(member_t *m)
{
    u64 next = log_next_index(&m->log);
    for (u32 s = 0; s < m->n_members; s++) {
        m->peers[s].next_index = next;
        m->peers[s].match_index = 0;
        m->peers[s].commit_index_sent = 0;
        m->peers[s].query_index = 0;
        m->peers[s].status = RA_PEER_NORMAL;
    }
}

/* ------------------------------------------------------------------ */
/* elections                                                           */
/* ------------------------------------------------------------------ */

/* call_for_election/3 :2853-2897 */
static u8 call_for_election(ctx_t *c, u8 target, nextq_t *nq)
{
    member_t *m = c->m;
    u64 last_idx, last_term; last_idx_term(m, &last_idx, &last_term);
    msg_t self; memset(&self, 0, sizeof self);
    msg_t req; memset(&req, 0, sizeof req);
    if (target == RA_CANDIDATE) {
        u64 new_term = m->current_term + 1;
        c->cnt->elections++;                                     /* :2856 */
        req.type = RA_EV_REQUEST_VOTE; req.term = new_term; req.a = last_idx; req.b = last_term;
        self.type = RA_EV_REQUEST_VOTE_RES; self.term = new_term; self.d = 1;
        update_term_and_voted_for(c, new_term, m->self_slot);
    } else {
        u64 token = ++m->token_counter;                          /* make_ref() */
        c->cnt->pre_vote_elections++;                            /* :2878 */
        req.type = RA_EV_PRE_VOTE; req.term = m->current_term; req.a = last_idx; req.b = last_term;
        req.c = token; req.d = (u64)1 /* ?RA_PROTO_VERSION */ | ((u64)m->machine_version << 32);
        self.type = RA_EV_PRE_VOTE_RES; self.term = m->current_term; self.c = token; self.d = 1;
        update_term_and_voted_for(c, m->current_term, m->self_slot);
        m->pre_vote_token = token;
    }
    m->leader_slot = RA_NO_SLOT;
    m->votes = 0;
    self.row = m->row; self.from_slot = m->self_slot;
    next_event(nq, &self, 0);                                    /* {next_event, cast, VoteForSelf} */
    for (u32 s = 0; s < m->n_members; s++) {                     /* {send_vote_requests, Reqs} */
        if (s == m->self_slot) continue;
        msg_t r = req; emit_msg(c, s, &r);
    }
    return target;
}

/* process_pre_vote/3 :2899-2956 */
static u8 process_pre_vote(ctx_t *c, u8 fsm_state, const msg_t *rpc)
{
    member_t *m = c->m;
    u64 term = rpc->term, token = rpc->c;
    u32 version = (u32)(rpc->d & 0xffffffffu), their_macver = (u32)(rpc->d >> 32);
    if (term >= m->current_term) {
        update_term(c, term);
        u64 li, lt; last_idx_term(m, &li, &lt);
        if (is_candidate_log_up_to_date(rpc->a, rpc->b, li, lt)) {
            if (version > 1) {                                               /* :2914-2917 */
                reply_vote_result(c, rpc->from_slot, RA_EV_PRE_VOTE_RES, term, token, 0);
            } else if (their_macver == m->effective_machine_version ||
                       (their_macver >= m->effective_machine_version &&
                        their_macver <= m->machine_version)) {              /* :2918-2928 */
                reply_vote_result(c, rpc->from_slot, RA_EV_PRE_VOTE_RES, term, token, 1);
            } else {                                                         /* :2929-2934 */
                reply_vote_result(c, rpc->from_slot, RA_EV_PRE_VOTE_RES, term, token, 0);
                c->status |= RA_ST_START_ELECTION_TMO;
            }
        } else if (fsm_state == RA_FOLLOWER) {                               /* :2941-2942 */
            c->status |= RA_ST_START_ELECTION_TMO;
        } else {                                                             /* :2943-2945 */
            reply_vote_result(c, rpc->from_slot, RA_EV_PRE_VOTE_RES, term, token, 0);
        }
    } else {                                                                 /* :2948-2956 */
        reply_vote_result(c, rpc->from_slot, RA_EV_PRE_VOTE_RES, m->current_term, token, 0);
    }
    return fsm_state;
}

/* ------------------------------------------------------------------ */
/* has_log_entry_or_snapshot/3 :3141-3156                               */
/* ------------------------------------------------------------------ */
enum { ENTRY_OK = 0, ENTRY_MISSING = 1, ENTRY_TERM_MISMATCH = 2 };
static int has_log_entry_or_snapshot(const member_t *m, u64 idx, u64 term)
{
    u64 t = log_fetch_term(&m->log, (i64)idx);
    if (t == UNDEF) {
        u64 si, st;
        if (log_snapshot(&m->log, &si, &st) && si == idx)
            return st == term ? ENTRY_OK : ENTRY_TERM_MISMATCH;
        return ENTRY_MISSING;
    }
    return t == term ? ENTRY_OK : ENTRY_TERM_MISMATCH;
}

/* term of the k-th entry of an AER record (see ra_event layout) */
static u64 aer_entry_term(const msg_t *e, u64 idx)
{
    if (e->n1 != 0 && idx - (e->a + 1) >= e->n1) return e->e;
    return e->d;
}

/* ------------------------------------------------------------------ */
/* handle_follower/2 :1264-1641                                         */
/* ------------------------------------------------------------------ */
static u8 handle_follower(ctx_t *c, const msg_t *e, nextq_t *nq)
{
    member_t *m = c->m;
    switch (e->type) {
    case RA_EV_AER: {
        u64 term = e->term, cur = m->current_term;
        u32 leader = e->from_slot;
        c->cnt->aer_received_follower++;                                     /* :1278 and :1418 */
        if (term >= cur) {                                                   /* :1266-1414 */
            u64 pl_idx = e->a, pl_term = e->b, leader_commit = e->c;
            c->status |= RA_ST_LEADER_MSG;                                   /* {record_leader_msg,_} */
            m->leader_slot = (u8)leader;
            update_term(c, term);
            int r = has_log_entry_or_snapshot(m, pl_idx, pl_term);
            if (r == ENTRY_OK) {
                /* drop_existing/3 :3673-3681 */
                u64 n0 = e->n, k = 0, last_valid = pl_idx;
                while (k < n0) {
                    u64 idx = pl_idx + 1 + k;
                    if (!log_exists(&m->log, idx, aer_entry_term(e, idx))) break;
                    last_valid = idx; k++;
                }
                if (k == n0) {                                               /* Entries == [] :1288 */
                    c->cnt->aer_received_follower_empty++;                   /* :1290 */
                    u64 local_last = m->log.last_index;
                    int validated;
                    if (n0 == 0 && local_last > pl_idx) {                    /* :1294-1303 */
                        if (pl_idx < m->last_applied) { set_fatal(c, RA_FATAL_ASSERT); return RA_FOLLOWER; }
                        if (!log_set_last_index(&m->log, pl_idx)) {
                            set_fatal(c, RA_FATAL_SET_LAST_INDEX_NOT_FOUND); return RA_FOLLOWER;
                        }
                        note(c, RA_NOTE_TRUNCATE, 0, m->log.last_index, m->log.last_term, 0);
                        validated = 1;
                    } else {
                        validated = local_last <= last_valid;                /* :1310 */
                    }
                    if (validated) {                                         /* :1313-1326 */
                        m->commit_index = leader_commit;
                        evaluate_commit_index_follower(c);
                        cast_reply(c, leader, make_aer_reply(m, term, 1));
                        return RA_FOLLOWER;
                    } else {                                                 /* :1327-1346 */
                        u64 lvi = m->last_applied > last_valid ? m->last_applied : last_valid;
                        msg_t rp; memset(&rp, 0, sizeof rp);
                        rp.type = RA_EV_AER_REPLY;
                        rp.term = cur;                                       /* CurTerm: the pre-update term */
                        rp.a = lvi + 1; rp.b = lvi; rp.c = srv_fetch_term(m, (i64)lvi); rp.d = 1;
                        cast_reply(c, leader, rp);
                        return RA_FOLLOWER;
                    }
                } else {                                                     /* [{FstIdx,_,_}|_] :1348-1371 */
                    u64 fst = pl_idx + 1 + k;
                    if (fst < m->last_applied) { set_fatal(c, RA_FATAL_ASSERT); return RA_FOLLOWER; }
                    /* ra_log:write/2 guard ra_log.erl:547-550 */
                    int empty = !(m->log.first_index <= m->log.last_index);
                    if (!empty && !(fst <= m->log.last_index + 1)) {
                        set_fatal(c, RA_FATAL_WRITE_INTEGRITY); return RA_FOLLOWER;
                    }
                    if (empty && !(fst == m->log.last_index + 1)) {
                        /* range undefined: production accepts any FstIdx; the engine's view
                           needs contiguity with the snapshot (ra_log_memory.erl:100-102) */
                        set_fatal(c, RA_FATAL_WRITE_INTEGRITY); return RA_FOLLOWER;
                    }
                    m->commit_index = leader_commit;                         /* :1349 */
                    if (fst <= m->log.last_index)                            /* truncating overwrite */
                        log_truncate(&m->log, fst - 1,
                                     fst == 0 ? 0 : (log_fetch_term(&m->log, (i64)fst - 1) != UNDEF
                                                     ? log_fetch_term(&m->log, (i64)fst - 1)
                                                     : m->log.snap_term));
                    u64 run_from = fst, run_term = aer_entry_term(e, fst);
                    for (u64 idx = fst; idx <= pl_idx + n0; idx++) {
                        u64 t = aer_entry_term(e, idx);
                        if (t != run_term) {
                            note(c, RA_NOTE_WAL_APPEND, 0, run_from, idx - 1, run_term);
                            run_from = idx; run_term = t;
                        }
                        log_push(&m->log, idx, t);
                    }
                    note(c, RA_NOTE_WAL_APPEND, 0, run_from, pl_idx + n0, run_term);
                    evaluate_commit_index_follower(c);
                    return RA_FOLLOWER;
                }
            } else if (r == ENTRY_MISSING) {                                 /* :1373-1387 */
                msg_t rp = make_aer_reply(m, term, 0);
                m->condition = 1; m->cond_reply_valid = 1;
                m->cond_reply_term = rp.term; m->cond_reply_next = rp.a;
                m->cond_reply_last_index = rp.b; m->cond_reply_last_term = rp.c;
                cast_reply(c, leader, rp);
                return RA_AWAIT_CONDITION;
            } else {                                                         /* term_mismatch :1388-1413 */
                /* mismatch_append_entries_reply/3 :3587-3595 */
                u64 la = m->last_applied;
                u64 lat = srv_fetch_term(m, (i64)la);
                if (lat == UNDEF) { set_fatal(c, RA_FATAL_ASSERT); return RA_FOLLOWER; }
                msg_t rp; memset(&rp, 0, sizeof rp);
                rp.type = RA_EV_AER_REPLY; rp.term = term; rp.a = la + 1; rp.b = la; rp.c = lat; rp.d = 0;
                m->condition = 2; m->cond_reply_valid = 1;
                m->cond_reply_term = rp.term; m->cond_reply_next = rp.a;
                m->cond_reply_last_index = rp.b; m->cond_reply_last_term = rp.c;
                cast_reply(c, leader, rp);
                return RA_AWAIT_CONDITION;
            }
        }
        /* :1415-1424 term lower than current */
        cast_reply(c, leader, make_aer_reply(m, cur, 0));
        return RA_FOLLOWER;
    }
    case RA_EV_WRITTEN: {                                                    /* :1441-1458 */
        u64 lwi = m->log.lw_idx, lwt = m->log.lw_term;
        log_handle_written(&m->log, e->term, e->a, e->b);
        if ((lwi != m->log.lw_idx || lwt != m->log.lw_term) && m->leader_slot != RA_NO_SLOT)
            cast_reply(c, m->leader_slot, make_aer_reply(m, m->current_term, 1));
        return RA_FOLLOWER;
    }
    case RA_EV_PRE_VOTE:                                                     /* :1459-1466 */
        if (m->membership != RA_VOTER) return RA_FOLLOWER;
        return process_pre_vote(c, RA_FOLLOWER, e);
    case RA_EV_REQUEST_VOTE: {                                               /* :1467-1513 */
        if (m->membership != RA_VOTER) return RA_FOLLOWER;
        u64 term = e->term, cur = m->current_term;
        u8 cand = e->from_slot;
        if (term == cur && m->voted_for != RA_NO_SLOT && m->voted_for != cand) {   /* :1473-1481 */
            reply_vote_result(c, cand, RA_EV_REQUEST_VOTE_RES, term, 0, 0);
            return RA_FOLLOWER;
        }
        if (term >= cur) {                                                   /* :1482-1505 */
            update_term(c, term);
            u64 li, lt; last_idx_term(m, &li, &lt);
            if (is_candidate_log_up_to_date(e->a, e->b, li, lt)) {
                reply_vote_result(c, cand, RA_EV_REQUEST_VOTE_RES, term, 0, 1);
                update_term_and_voted_for(c, term, cand);
            } else {
                reply_vote_result(c, cand, RA_EV_REQUEST_VOTE_RES, term, 0, 0);
            }
            return RA_FOLLOWER;
        }
        reply_vote_result(c, cand, RA_EV_REQUEST_VOTE_RES, cur, 0, 0);       /* :1506-1513 */
        return RA_FOLLOWER;
    }
    case RA_EV_AER_REPLY: {                                                  /* :1514-1517 */
        u64 t = e->term > m->current_term ? e->term : m->current_term;
        update_term(c, t);
        return RA_FOLLOWER;
    }
    case RA_EV_ELECTION_TIMEOUT:                                             /* :1603-1610 */
        if (m->membership != RA_VOTER) return RA_FOLLOWER;
        return call_for_election(c, RA_PRE_VOTE, nq);
    case RA_EV_COMMAND:                       /* ra_server_proc.erl:827-845: redirect / reject */
        note(c, RA_NOTE_NOT_LEADER, 0, e->n, m->leader_slot, 0);
        return RA_FOLLOWER;
    case RA_EV_CONSISTENT_QUERY:              /* only a leader answers consistent queries */
        note(c, RA_NOTE_NOT_LEADER, 0, 0, m->leader_slot, 0);
        return RA_FOLLOWER;
    case RA_EV_HEARTBEAT_RPC:
        if (e->term >= m->current_term) {                                    /* :1425-1434 */
            update_term(c, e->term);
            m->leader_slot = e->from_slot;
            send_heartbeat_reply(c, e->from_slot, e->term, e->a);
        } else {                                                             /* :1435-1440 */
            send_heartbeat_reply(c, e->from_slot, m->current_term, e->a);
        }
        return RA_FOLLOWER;
    case RA_EV_HEARTBEAT_REPLY:                                              /* :1518-1521 */
        update_term(c, e->term > m->current_term ? e->term : m->current_term);
        return RA_FOLLOWER;
    default:                                  /* :1593-1602, :1639-1641 */
        return RA_FOLLOWER;
    }
}

/* ------------------------------------------------------------------ */
/* handle_leader/2 :520-1023                                            */
/* ------------------------------------------------------------------ */
static void pipeline_next_event(nextq_t *nq, const member_t *m)
{
    msg_t p; memset(&p, 0, sizeof p);
    p.type = RA_EV_PIPELINE_RPCS; p.row = m->row; p.from_slot = RA_NO_SLOT;
    next_event(nq, &p, 1);                                   /* {next_event, info, pipeline_rpcs} */
}

static u8 step_down(ctx_t *c, u64 term)
{   /* {follower, update_term(Term, State0#{leader_id => undefined}), _} */
    c->m->leader_slot = RA_NO_SLOT;
    update_term(c, term);
    return RA_FOLLOWER;
}

static u8 handle_leader(ctx_t *c, const msg_t *e, nextq_t *nq, int pure)
{
    member_t *m = c->m;
    switch (e->type) {
    case RA_EV_AER_REPLY: {
        u64 term = e->term;
        u32 from = e->from_slot;
        int success = e->d != 0;
        if (success && term == m->current_term) {                            /* :522-561 */
            c->cnt->aer_replies_success++;                                   /* :528 */
            if (!is_peer(m, from)) return RA_LEADER;
            peer_t *p = &m->peers[from];
            if (e->b > p->match_index) p->match_index = e->b;                /* max(MI, LastIdx) */
            if (e->a > p->next_index) p->next_index = e->a;                  /* max(NI, NextIdx) */
            evaluate_quorum(c);
            pipeline_next_event(nq, m);
            return RA_LEADER;
        }
        if (term > m->current_term) {                                        /* :562-576 */
            if (!is_peer(m, from)) return RA_LEADER;
            return step_down(c, term);
        }
        if (!success) {                                                      /* :577-643 */
            if (!is_peer(m, from)) return RA_LEADER;
            c->cnt->aer_replies_failed++;                                    /* :590 */
            peer_t *p = &m->peers[from];
            u64 peer_next = e->a, peer_last = e->b, peer_last_term = e->c;
            u64 mi = p->match_index, ni = p->next_index;
            u64 t = log_fetch_term(&m->log, (i64)peer_last);
            if (t == UNDEF) {                                                /* :596-601 */
                p->next_index = peer_next;
            } else if (t == peer_last_term && peer_last >= mi) {             /* :603-610 */
                p->match_index = peer_last; p->next_index = peer_next;
            } else if (peer_last < mi) {                                     /* :611-622 */
                p->match_index = peer_last; p->next_index = peer_last + 1;
            } else {                                                         /* :623-639 */
                i64 a = (i64)ni - 1, b = (i64)peer_next;
                i64 x = a < b ? a : b;
                p->next_index = x > (i64)mi ? (u64)x : mi;
            }
            (void)make_pipelined_rpc_effects(c, 0, pure);
            return RA_LEADER;
        }
        return RA_LEADER;                                   /* stale success: unhandled :1021 */
    }
    case RA_EV_COMMAND: {                                                    /* :644-729 */
        u64 n = e->n;
        int noop = (e->flags & RA_EVF_NOOP) != 0;
        if (n == 0) return RA_LEADER;
        u64 from = log_next_index(&m->log);
        for (u64 k = 0; k < n; k++)                                          /* append_log_leader/3 :3516-3523 */
            log_push(&m->log, log_next_index(&m->log), m->current_term);
        note(c, RA_NOTE_WAL_APPEND, 0, from, from + n - 1, m->current_term);
        (void)make_pipelined_rpc_effects(c, noop, pure);
        return RA_LEADER;
    }
    case RA_EV_WRITTEN:                                                      /* :730-735 */
        log_handle_written(&m->log, e->term, e->a, e->b);
        evaluate_quorum(c);
        pipeline_next_event(nq, m);
        return RA_LEADER;
    case RA_EV_PIPELINE_RPCS:                                                /* :784-792 */
        if (make_pipelined_rpc_effects(c, 0, pure)) pipeline_next_event(nq, m);
        return RA_LEADER;
    case RA_EV_AER: {
        if (e->term > m->current_term) {                                     /* :826-835 */
            u8 r = step_down(c, e->term);
            next_event(nq, e, 0);
            return r;
        }
        if (e->term == m->current_term) {                                    /* :836-840 */
            set_fatal(c, RA_FATAL_LEADER_SAW_AER_SAME_TERM);
            return RA_LEADER;
        }
        cast_reply(c, e->from_slot, make_aer_reply(m, m->current_term, 0));  /* :841-845 */
        return RA_LEADER;
    }
    case RA_EV_REQUEST_VOTE:
        if (e->term > m->current_term) {                                     /* :919-933 */
            if (!is_peer(m, e->from_slot)) return RA_LEADER;
            u8 r = step_down(c, e->term);
            next_event(nq, e, 0);
            return r;
        }
        reply_vote_result(c, e->from_slot, RA_EV_REQUEST_VOTE_RES, m->current_term, 0, 0);  /* :934-936 */
        return RA_LEADER;
    case RA_EV_PRE_VOTE:
        if (e->term > m->current_term) {                                     /* :937-951 */
            if (!is_peer(m, e->from_slot)) return RA_LEADER;
            u8 r = step_down(c, e->term);
            next_event(nq, e, 0);
            return r;
        }
        make_rpcs(c, 1);                                    /* enforce leadership :952-957 */
        return RA_LEADER;
    case RA_EV_TICK:                                        /* ra_server_proc.erl:610-613 */
        make_rpcs(c, 0);
        return RA_LEADER;
    case RA_EV_CONSISTENT_QUERY:                            /* :846-851 + make_heartbeat_rpc_effects/2 :3722-3739 */
        if (m->n_members <= 1) {                            /* no peers: apply right away */
            note(c, RA_NOTE_QUERY_APPLY, 0, m->commit_index, 0, 0);
            return RA_LEADER;
        }
        m->query_index++;
        heartbeat_rpc_effects(c, m->query_index);
        note(c, RA_NOTE_QUERY_INDEX, 0, m->query_index, m->commit_index, 0);
        return RA_LEADER;
    case RA_EV_HEARTBEAT_RPC:
        if (e->term > m->current_term) {                                     /* :871-880 */
            u8 r = step_down(c, e->term);
            next_event(nq, e, 0);
            return r;
        }
        if (e->term < m->current_term) {                                     /* :881-888 */
            send_heartbeat_reply(c, e->from_slot, m->current_term, e->a);
            return RA_LEADER;
        }
        set_fatal(c, RA_FATAL_LEADER_SAW_HEARTBEAT_SAME_TERM);               /* :889-894 */
        return RA_LEADER;
    case RA_EV_HEARTBEAT_REPLY:                                              /* :895-918 */
        if (e->term == m->current_term) {                   /* heartbeat_rpc_quorum/3 :3773-3795 */
            if (is_peer(m, e->from_slot) && e->a > m->peers[e->from_slot].query_index)
                m->peers[e->from_slot].query_index = e->a;
            query_agreed(c, query_quorum(m));
            return RA_LEADER;
        }
        if (e->term > m->current_term) return step_down(c, e->term);
        return RA_LEADER;                                   /* lower term: ignored */
    default:                                                /* :958-963, :1021-1023 */
        return RA_LEADER;
    }
}

/* ------------------------------------------------------------------ */
/* handle_candidate/2 :1026-1171                                        */
/* ------------------------------------------------------------------ */
static u8 handle_candidate(ctx_t *c, const msg_t *e, nextq_t *nq)
{
    member_t *m = c->m;
    switch (e->type) {
    case RA_EV_REQUEST_VOTE_RES:
        if (e->d && e->term == m->current_term) {                            /* :1028-1044 */
            u32 nv = m->votes + 1;
            if (nv == required_quorum(m)) {
                m->leader_slot = m->self_slot;
                initialise_peers(m);
                m->votes = 0;                                   /* maps:without([votes], State) */
                /* post_election_effects/1 :4001-4037: noop with the effective machine version */
                msg_t nop; memset(&nop, 0, sizeof nop);
                nop.type = RA_EV_COMMAND; nop.flags = RA_EVF_NOOP; nop.n = 1;
                nop.row = m->row; nop.from_slot = RA_NO_SLOT;
                next_event(nq, &nop, 0);
                c->cnt->elections_won++;
                return RA_LEADER;
            }
            m->votes = nv;
            return RA_CANDIDATE;
        }
        if (e->term > m->current_term) {                                     /* :1045-1052 */
            update_term_and_voted_for(c, e->term, RA_NO_SLOT);
            return RA_FOLLOWER;
        }
        return RA_CANDIDATE;                                                 /* :1053-1054, :1115 */
    case RA_EV_AER:
        if (e->term >= m->current_term) {                                    /* :1055-1058 */
            update_term_and_voted_for(c, e->term, RA_NO_SLOT);
            next_event(nq, e, 0);
            return RA_FOLLOWER;
        }
        cast_reply(c, e->from_slot, make_aer_reply(m, m->current_term, 0));  /* :1059-1063 */
        return RA_CANDIDATE;
    case RA_EV_AER_REPLY:
        if (e->term > m->current_term) {                                     /* :1082-1090 */
            update_term_and_voted_for(c, e->term, RA_NO_SLOT);
            return RA_FOLLOWER;
        }
        return RA_CANDIDATE;
    case RA_EV_REQUEST_VOTE:
        if (e->term > m->current_term) {                                     /* :1091-1098 */
            update_term_and_voted_for(c, e->term, RA_NO_SLOT);
            next_event(nq, e, 0);
            return RA_FOLLOWER;
        }
        reply_vote_result(c, e->from_slot, RA_EV_REQUEST_VOTE_RES, m->current_term, 0, 0);  /* :1107-1109 */
        return RA_CANDIDATE;
    case RA_EV_PRE_VOTE:
        if (e->term > m->current_term) {                                     /* :1099-1106 */
            update_term_and_voted_for(c, e->term, RA_NO_SLOT);
            next_event(nq, e, 0);
            return RA_FOLLOWER;
        }
        return process_pre_vote(c, RA_CANDIDATE, e);                         /* :1110-1114 */
    case RA_EV_WRITTEN:                                                      /* :1140-1143 */
        log_handle_written(&m->log, e->term, e->a, e->b);
        return RA_CANDIDATE;
    case RA_EV_ELECTION_TIMEOUT:                                             /* :1144-1145 */
        return call_for_election(c, RA_CANDIDATE, nq);
    case RA_EV_COMMAND:                                     /* ra_server_proc.erl:680-684 reject */
        note(c, RA_NOTE_NOT_LEADER, 0, e->n, m->leader_slot, 0);
        return RA_CANDIDATE;
    case RA_EV_CONSISTENT_QUERY:
        note(c, RA_NOTE_NOT_LEADER, 0, 0, m->leader_slot, 0);
        return RA_CANDIDATE;
    case RA_EV_HEARTBEAT_RPC:
        if (e->term >= m->current_term) {                                    /* :1064-1067 */
            update_term_and_voted_for(c, e->term, RA_NO_SLOT);
            next_event(nq, e, 0);
            return RA_FOLLOWER;
        }
        send_heartbeat_reply(c, e->from_slot, m->current_term, e->a);        /* :1068-1073 */
        return RA_CANDIDATE;
    case RA_EV_HEARTBEAT_REPLY:
        if (e->term > m->current_term) {                                     /* :1074-1081 */
            update_term_and_voted_for(c, e->term, RA_NO_SLOT);
            return RA_FOLLOWER;
        }
        return RA_CANDIDATE;
    default:
        return RA_CANDIDATE;
    }
}

/* ------------------------------------------------------------------ */
/* handle_pre_vote/2 :1173-1261                                         */
/* ------------------------------------------------------------------ */
static u8 handle_pre_vote(ctx_t *c, const msg_t *e, nextq_t *nq)
{
    member_t *m = c->m;
    switch (e->type) {
    case RA_EV_AER:
        if (e->term >= m->current_term) {                                    /* :1175-1180 */
            update_term(c, e->term);
            m->votes = 0;
            next_event(nq, e, 0);
            return RA_FOLLOWER;
        }
        return RA_PRE_VOTE;                                 /* unhandled :1259 */
    case RA_EV_REQUEST_VOTE:
        if (e->term > m->current_term) {                                     /* :1196-1201 */
            update_term(c, e->term);
            m->votes = 0;
            next_event(nq, e, 0);
            return RA_FOLLOWER;
        }
        return RA_PRE_VOTE;                                 /* unhandled :1259 */
    case RA_EV_PRE_VOTE_RES:
        if (e->term > m->current_term) {                                     /* :1202-1207 */
            update_term(c, e->term);
            m->votes = 0;
            return RA_FOLLOWER;
        }
        if (e->d && e->term == m->current_term && e->c == m->pre_vote_token &&
            m->membership == RA_VOTER) {                                     /* :1212-1229 */
            u32 nv = m->votes + 1;
            if (nv == required_quorum(m)) return call_for_election(c, RA_CANDIDATE, nq);
            m->votes = nv;
            return RA_PRE_VOTE;
        }
        return RA_PRE_VOTE;                                                  /* :1230-1232 */
    case RA_EV_PRE_VOTE:                                                     /* :1233-1234 */
        return process_pre_vote(c, RA_PRE_VOTE, e);
    case RA_EV_ELECTION_TIMEOUT:                                             /* :1238-1239 */
        return call_for_election(c, RA_PRE_VOTE, nq);
    case RA_EV_WRITTEN:                                                      /* :1240-1243 */
        log_handle_written(&m->log, e->term, e->a, e->b);
        return RA_PRE_VOTE;
    case RA_EV_COMMAND:                                     /* ra_server_proc.erl:746-750 reject */
        note(c, RA_NOTE_NOT_LEADER, 0, e->n, m->leader_slot, 0);
        return RA_PRE_VOTE;
    case RA_EV_CONSISTENT_QUERY:
        note(c, RA_NOTE_NOT_LEADER, 0, 0, m->leader_slot, 0);
        return RA_PRE_VOTE;
    case RA_EV_HEARTBEAT_RPC:
        if (e->term >= m->current_term) {                                    /* :1181-1186 */
            update_term(c, e->term);
            m->votes = 0;
            next_event(nq, e, 0);
            return RA_FOLLOWER;
        }
        send_heartbeat_reply(c, e->from_slot, m->current_term, e->a);        /* :1187-1191 */
        return RA_PRE_VOTE;
    case RA_EV_HEARTBEAT_REPLY:
        if (e->term > m->current_term) {                                     /* :1192-1195 */
            m->votes = 0;
            update_term(c, e->term);
            return RA_FOLLOWER;
        }
        return RA_PRE_VOTE;
    default:
        return RA_PRE_VOTE;
    }
}

/* ------------------------------------------------------------------ */
/* handle_await_condition/2 :1900-1941 with follower_catchup_cond/3 :2184-2213 */
/* ------------------------------------------------------------------ */
static u8 handle_await_condition(ctx_t *c, const msg_t *e, nextq_t *nq)
{
    member_t *m = c->m;
    switch (e->type) {
    case RA_EV_REQUEST_VOTE:                                                 /* :1902-1903 */
        next_event(nq, e, 0);
        return RA_FOLLOWER;
    case RA_EV_PRE_VOTE:                                                     /* :1904-1905 */
        return process_pre_vote(c, RA_AWAIT_CONDITION, e);
    case RA_EV_ELECTION_TIMEOUT:                                             /* :1906-1913 */
        if (m->membership != RA_VOTER) return RA_AWAIT_CONDITION;
        return call_for_election(c, RA_PRE_VOTE, nq);
    case RA_EV_AWAIT_COND_TIMEOUT: {                                         /* :1914-1927 */
        /* the catch-up predicate answers false for this message (:2212-2213):
           repeat the stored reply effect and fall back to follower */
        if (m->cond_reply_valid && m->leader_slot != RA_NO_SLOT) {
            msg_t rp; memset(&rp, 0, sizeof rp);
            rp.type = RA_EV_AER_REPLY; rp.term = m->cond_reply_term; rp.a = m->cond_reply_next;
            rp.b = m->cond_reply_last_index; rp.c = m->cond_reply_last_term; rp.d = 0;
            cast_reply(c, m->leader_slot, rp);
            c->status |= RA_ST_LEADER_MSG;                  /* the repeated {record_leader_msg,_} */
        }
        m->condition = 0; m->cond_reply_valid = 0;
        return RA_FOLLOWER;
    }
    case RA_EV_WRITTEN:                                                      /* :1928-1931 */
        log_handle_written(&m->log, e->term, e->a, e->b);
        return RA_AWAIT_CONDITION;
    case RA_EV_AER: {                                                        /* :1932-1941 */
        int ok = 0;
        if (e->term >= m->current_term) {                                    /* :2184-2202 */
            int r = has_log_entry_or_snapshot(m, e->a, e->b);
            if (r == ENTRY_OK) ok = 1;
            else if (r == ENTRY_TERM_MISMATCH) ok = (m->condition == 1);     /* OriginalReason == missing */
        }
        if (ok) {
            m->condition = 0; m->cond_reply_valid = 0;
            next_event(nq, e, 0);
            return RA_FOLLOWER;
        }
        return RA_AWAIT_CONDITION;
    }
    case RA_EV_CONSISTENT_QUERY:
        note(c, RA_NOTE_NOT_LEADER, 0, 0, m->leader_slot, 0);
        return RA_AWAIT_CONDITION;
    case RA_EV_COMMAND:                                     /* ra_server_proc.erl:1144-1163 postponed */
        c->status |= RA_ST_CMD_POSTPONED;
        return RA_AWAIT_CONDITION;
    default:                                                /* predicate false :1938-1940 */
        return RA_AWAIT_CONDITION;
    }
}

/* ------------------------------------------------------------------ */
/* the ra_server_proc shim: dispatch, state enter, next_event chasing   */
/* ------------------------------------------------------------------ */
static u8 dispatch(ctx_t *c, const msg_t *e, nextq_t *nq, int pure)
{
    switch (c->m->role) {
    case RA_LEADER:          return handle_leader(c, e, nq, pure);
    case RA_FOLLOWER:        return handle_follower(c, e, nq);
    case RA_CANDIDATE:       return handle_candidate(c, e, nq);
    case RA_PRE_VOTE:        return handle_pre_vote(c, e, nq);
    case RA_AWAIT_CONDITION: return handle_await_condition(c, e, nq);
    default:                 return c->m->role;
    }
}

/* ra_server:handle_state_enter/3 -> become/3 :2153-2177 */
static void become(member_t *m, u8 new_role)
{
    if (new_role == RA_FOLLOWER)
        for (u32 s = 0; s < m->n_members; s++) m->peers[s].status = RA_PEER_NORMAL;
}

static void emit_next_event_record(ctx_t *c, const msg_t *e)
{
    msg_t r = *e;
    r.flags |= RA_EVF_NEXT_EVENT;
    emit_msg(c, c->m->self_slot, &r);
}

/* evaluate one input event of a row, chasing {next_event,_} like gen_statem does
   (ra_server_proc.erl:1574-1577: inserted ahead of the mailbox, in order)        */
static void process_event(ctx_t *c, const msg_t *in)
{
    member_t *m = c->m;
    int pure = c->o->cfg.pure != 0;
    msg_t pend[12]; u32 np = 0;
    pend[np++] = *in;
    int pipeline_chased = 0;
    c->cnt->events++;
    while (np > 0) {
        if (m->fatal) return;
        msg_t e = pend[0];
        memmove(pend, pend + 1, (--np) * sizeof(msg_t));
        if (e.type == RA_EV_PIPELINE_RPCS && (e.flags & RA_EVF_INFO)) {
            /* contract: one chased pipeline pass per input event, the rest next step */
            if (pipeline_chased) { m->pipeline_pending = 1; c->status |= RA_ST_PIPELINE_PENDING; continue; }
            pipeline_chased = 1;
        }
        nextq_t nq; nq.n = 0;
        u8 old = m->role;
        u8 nr = dispatch(c, &e, &nq, pure);
        if (m->fatal) return;
        if (nr != old) {
            m->role = nr;
            c->status |= RA_ST_ROLE_CHANGED;
            if (!pure) become(m, nr);
            if (nr == RA_LEADER) c->status |= RA_ST_BECAME_LEADER;
        }
        if (pure) {
            for (u32 i = 0; i < nq.n; i++) emit_next_event_record(c, &nq.q[i]);
            continue;
        }
        /* candidate -> leader: the proc puts tick_timeout ahead of the effects' next
           events (ra_server_proc.erl:728-730) */
        msg_t front[8]; u32 nf = 0;
        if (nr == RA_LEADER && old == RA_CANDIDATE) {
            msg_t t; memset(&t, 0, sizeof t);
            t.type = RA_EV_TICK; t.row = m->row; t.from_slot = RA_NO_SLOT;
            front[nf++] = t;
        }
        for (u32 i = 0; i < nq.n && nf < 8; i++) front[nf++] = nq.q[i];
        if (nf) {
            if (np + nf > 12) nf = 12 - np;
            memmove(pend + nf, pend, np * sizeof(msg_t));
            memcpy(pend, front, nf * sizeof(msg_t));
            np += nf;
        }
    }
}

static void ctx_begin(ctx_t *c, ra_oracle *o, member_t *m, ra_counters *cnt, int routed_out)
{
    memset(c, 0, sizeof *c);
    c->o = o; c->m = m; c->cnt = cnt; c->routed_out = routed_out;
    c->role_at_start = m->role;
}

/* end of a row's step: the STATUS note */
static void ctx_finish(ctx_t *c)
{
    member_t *m = c->m;
    if (c->status == 0) return;
    if (c->status == RA_ST_LEADER_MSG && c->n_notes > 0) {   /* rides in the aux of the row's last note */
        c->notes[c->n_notes - 1].aux = (uint16_t)c->status;
        return;
    }
    ra_note *n = &c->notes[c->n_notes++];           /* one slot is always reserved */
    n->row = m->row; n->type = RA_NOTE_STATUS; n->slot = m->self_slot; n->aux = (uint16_t)c->status;
    n->a = m->current_term;
    n->b = (u64)m->voted_for | ((u64)m->leader_slot << 8) | ((u64)c->role_at_start << 16) |
           ((u64)m->role << 24);
    n->c = c->fatal_code | ((u64)c->unconsumed << 8);
    if (c->status & RA_ST_FATAL) c->cnt->fatal_rows++;
}

/* inputs of a row that do not come from the caller: deferred pipeline pass, mailboxes */
static void process_row_prologue(ctx_t *c)
{
    ra_oracle *o = c->o; member_t *m = c->m;
    if (m->pipeline_pending) {
        m->pipeline_pending = 0;
        msg_t p; memset(&p, 0, sizeof p);
        p.type = RA_EV_PIPELINE_RPCS; p.row = m->row; p.from_slot = RA_NO_SLOT;
        process_event(c, &p);
    }
    if (o->cfg.route_on_device) {
        int cb = o->cur;
        for (u32 s = 0; s < m->n_members; s++) {
            u8 *cnt = &o->mbox_n[cb][(size_t)s * o->n_rows + m->row];
            for (u32 k = 0; k < *cnt; k++)
                take_record(c, &o->mbox[cb][((size_t)s * RA_MBOX_DEPTH + k) * o->n_rows + m->row]);
            *cnt = 0;
        }
    }
}

static void publish_mbox_counts(ctx_t *c)
{
    ra_oracle *o = c->o; member_t *m = c->m;
    if (!o->cfg.route_on_device) return;
    int nb = o->cur ^ 1;
    u32 g = group_of(o, m->row);
    for (u32 s = 0; s < m->n_members; s++) {
        if (s == m->self_slot) continue;
        o->mbox_n[nb][(size_t)m->self_slot * o->n_rows + row_of(o, g, s)] = c->sent_to[s];
    }
}

/* ------------------------------------------------------------------ */
/* public API                                                          */
/* ------------------------------------------------------------------ */
static void member_init_empty(ra_oracle *o, member_t *m, u32 row)
{
    /* ra_server_SUITE:empty_state/2 :4022-4032 = ra_server:init/1 on a fresh
       ra_log_memory: entries #{0 => {0,undefined}}, last_written {0,0}, term 0 */
    u64 *keep = m->log.terms; size_t cap = m->log.store_cap;
    memset(m, 0, sizeof *m);
    m->log.terms = keep; m->log.store_cap = cap;
    m->row = row;
    m->self_slot = (u8)(row / o->cfg.n_groups);
    m->n_members = (u8)o->cfg.n_members;
    m->role = RA_FOLLOWER;
    m->leader_slot = RA_NO_SLOT; m->voted_for = RA_NO_SLOT;
    m->membership = RA_VOTER;
    for (u32 s = 0; s < m->n_members; s++) {
        m->peers[s].next_index = 1; m->peers[s].match_index = 0;
        m->peers[s].commit_index_sent = 0; m->peers[s].status = RA_PEER_NORMAL;
        m->peers[s].voter = 1;
    }
    m->log.first_index = 0; m->log.last_index = 0; m->log.last_term = 0;
    m->log.store_base = 0;
    log_reserve(&m->log, 0);
    m->log.store_base = 0;
    m->log.terms[0] = 0;
    m->log.n_runs = 1;
}

int ra_oracle_create(const ra_engine_cfg *cfg, ra_oracle **out)
{
    if (!cfg || !out || cfg->n_members < 1 || cfg->n_members > RA_MAX_MEMBERS || cfg->n_groups == 0)
        return RA_E_INVAL;
    if (cfg->n_shards > 1) return RA_E_INVAL;      /* the oracle is the unsharded truth */
    ra_oracle *o = (ra_oracle *)calloc(1, sizeof *o);
    if (!o) return RA_E_NOMEM;
    o->cfg = *cfg;
    if (cfg->note_cap && (cfg->note_cap < RA_NOTE_RESERVE + 2 || cfg->note_cap > RA_NOTE_CAP)) { free(o); return RA_E_INVAL; }
    o->note_cap = cfg->note_cap ? cfg->note_cap : RA_NOTE_CAP;
    if (o->cfg.max_pipeline_count == 0) o->cfg.max_pipeline_count = 4096;
    if (o->cfg.max_aer_batch == 0) o->cfg.max_aer_batch = 128;
    o->n_rows = cfg->n_groups * cfg->n_members;
    o->m = (member_t *)calloc(o->n_rows, sizeof(member_t));
    if (!o->m) { free(o); return RA_E_NOMEM; }
    if (cfg->route_on_device) {
        for (int b = 0; b < 2; b++) {
            o->mbox[b] = (ra_event *)calloc((size_t)cfg->n_members * RA_MBOX_DEPTH * o->n_rows, sizeof(ra_event));
            o->mbox_n[b] = (u8 *)calloc((size_t)cfg->n_members * o->n_rows, 1);
        }
        o->loc = (ra_event *)calloc((size_t)RA_LOCAL_CAP * o->n_rows, sizeof(ra_event));
        o->loc_n = (u8 *)calloc(o->n_rows, 1);
    }
    for (u32 r = 0; r < o->n_rows; r++) member_init_empty(o, &o->m[r], r);
    *out = o;
    return RA_OK;
}

void ra_oracle_destroy(ra_oracle *o)
{
    if (!o) return;
    for (u32 r = 0; r < o->n_rows; r++) free(o->m[r].log.terms);
    for (int b = 0; b < 2; b++) { free(o->mbox[b]); free(o->mbox_n[b]); }
    free(o->loc); free(o->loc_n);
    free(o->m); free(o);
}

int ra_oracle_reset_empty(ra_oracle *o)
{
    for (u32 r = 0; r < o->n_rows; r++) member_init_empty(o, &o->m[r], r);
    memset(&o->cnt, 0, sizeof o->cnt);
    if (o->cfg.route_on_device) {
        for (int b = 0; b < 2; b++) memset(o->mbox_n[b], 0, (size_t)o->cfg.n_members * o->n_rows);
        memset(o->loc_n, 0, o->n_rows);
    }
    o->step_no = 0;
    return RA_OK;
}

int ra_oracle_load_rows(ra_oracle *o, const ra_row_state *rows, size_t n)
{
    for (size_t i = 0; i < n; i++) {
        const ra_row_state *s = &rows[i];
        if (s->row >= o->n_rows || s->n_members != o->cfg.n_members || !ra_row_state_valid(s)) return RA_E_INVAL;
        member_t *m = &o->m[s->row];
        member_init_empty(o, m, s->row);
        m->role = s->role; m->self_slot = s->self_slot; m->n_members = s->n_members;
        m->leader_slot = s->leader_slot; m->voted_for = s->voted_for; m->membership = s->membership;
        m->condition = s->condition; m->votes = s->votes;
        m->machine_version = s->machine_version;
        m->effective_machine_version = s->effective_machine_version;
        m->pipeline_pending = (s->flags & 1) != 0;
        m->cond_reply_valid = (s->flags & 2) != 0;
        m->current_term = s->current_term; m->commit_index = s->commit_index;
        m->last_applied = s->last_applied; m->pre_vote_token = s->pre_vote_token;
        m->token_counter = s->token_counter;
        m->cond_reply_term = s->cond_reply_term; m->cond_reply_next = s->cond_reply_next_index;
        m->cond_reply_last_index = s->cond_reply_last_index;
        m->cond_reply_last_term = s->cond_reply_last_term;
        for (u32 p = 0; p < RA_MAX_MEMBERS; p++) {
            m->peers[p].next_index = s->peers[p].next_index;
            m->peers[p].match_index = s->peers[p].match_index;
            m->peers[p].commit_index_sent = s->peers[p].commit_index_sent;
            m->peers[p].status = s->peers[p].status;
            m->peers[p].voter = s->peers[p].voter;
            m->peers[p].query_index = 0;
        }
        m->query_index = 0; m->agreed_index = 0;
        if (o->cfg.route_on_device)      /* a (re)loaded member starts with an empty mailbox */
            for (int b = 0; b < 2; b++)
                for (u32 p = 0; p < o->cfg.n_members; p++) o->mbox_n[b][(size_t)p * o->n_rows + s->row] = 0;
        log_t *l = &m->log;
        l->first_index = s->first_index; l->last_index = s->last_index; l->last_term = s->last_term;
        l->lw_idx = s->last_written_index; l->lw_term = s->last_written_term;
        l->has_snapshot = s->has_snapshot; l->snap_idx = s->snapshot_index; l->snap_term = s->snapshot_term;
        l->n_runs = s->n_runs;
        l->store_base = l->first_index;
        if (l->first_index <= l->last_index) {
            log_reserve(l, l->last_index);
            for (u32 r = 0; r < s->n_runs; r++) {
                u64 end = (r + 1 < s->n_runs) ? s->run_start[r + 1] - 1 : s->last_index;
                for (u64 i = s->run_start[r]; i <= end; i++) l->terms[i - l->store_base] = s->run_term[r];
            }
        }
    }
    return RA_OK;
}

int ra_oracle_load_query_state(ra_oracle *o, const ra_query_state *q, size_t n)
{
    if (!o || (!q && n)) return RA_E_INVAL;
    for (size_t i = 0; i < n; i++) if (q[i].row >= o->n_rows) return RA_E_INVAL;
    for (size_t i = 0; i < n; i++) {
        member_t *m = &o->m[q[i].row];
        m->query_index = q[i].query_index; m->agreed_index = q[i].agreed_index;
        for (u32 p = 0; p < RA_MAX_MEMBERS; p++) m->peers[p].query_index = q[i].peer_query_index[p];
    }
    return RA_OK;
}

int ra_oracle_read_query_state(ra_oracle *o, ra_query_state *q, size_t n)
{
    if (!o || (!q && n)) return RA_E_INVAL;
    for (size_t i = 0; i < n; i++) if (q[i].row >= o->n_rows) return RA_E_INVAL;
    for (size_t i = 0; i < n; i++) {
        const member_t *m = &o->m[q[i].row];
        q[i]._pad = 0; q[i].query_index = m->query_index; q[i].agreed_index = m->agreed_index;
        for (u32 p = 0; p < RA_MAX_MEMBERS; p++) q[i].peer_query_index[p] = p < m->n_members ? m->peers[p].query_index : 0;
    }
    return RA_OK;
}

int ra_oracle_read_rows(ra_oracle *o, ra_row_state *rows, size_t n)
{
    for (size_t i = 0; i < n; i++) {
        ra_row_state *s = &rows[i];
        u32 row = s->row;
        if (row >= o->n_rows) return RA_E_INVAL;
        const member_t *m = &o->m[row];
        memset(s, 0, sizeof *s);
        s->row = row; s->role = m->role; s->self_slot = m->self_slot; s->n_members = m->n_members;
        s->leader_slot = m->leader_slot; s->voted_for = m->voted_for; s->membership = m->membership;
        s->condition = m->condition; s->has_snapshot = m->log.has_snapshot; s->votes = m->votes;
        s->machine_version = m->machine_version;
        s->effective_machine_version = m->effective_machine_version;
        s->flags = (m->pipeline_pending ? 1u : 0u) | (m->cond_reply_valid ? 2u : 0u) | (m->fatal ? 4u : 0u);
        s->current_term = m->current_term; s->commit_index = m->commit_index;
        s->last_applied = m->last_applied; s->pre_vote_token = m->pre_vote_token;
        s->token_counter = m->token_counter;
        s->cond_reply_term = m->cond_reply_term; s->cond_reply_next_index = m->cond_reply_next;
        s->cond_reply_last_index = m->cond_reply_last_index;
        s->cond_reply_last_term = m->cond_reply_last_term;
        for (u32 p = 0; p < RA_MAX_MEMBERS; p++) {
            s->peers[p].next_index = m->peers[p].next_index;
            s->peers[p].match_index = m->peers[p].match_index;
            s->peers[p].commit_index_sent = m->peers[p].commit_index_sent;
            s->peers[p].status = m->peers[p].status;
            s->peers[p].voter = m->peers[p].voter;
        }
        const log_t *l = &m->log;
        s->first_index = l->first_index; s->last_index = l->last_index; s->last_term = l->last_term;
        s->last_written_index = l->lw_idx; s->last_written_term = l->lw_term;
        s->snapshot_index = l->snap_idx; s->snapshot_term = l->snap_term;
        u32 nr = 0;
        if (l->first_index <= l->last_index) {
            for (u64 idx = l->first_index; idx <= l->last_index; idx++) {
                u64 t = l->terms[idx - l->store_base];
                if (nr == 0 || s->run_term[nr - 1] != t) {
                    if (nr >= RA_MAX_RUNS) return RA_E_CAPACITY;
                    s->run_start[nr] = idx; s->run_term[nr] = t; nr++;
                }
            }
        }
        s->n_runs = nr;
    }
    return RA_OK;
}

typedef struct { u32 row; u32 first_msg, n_msgs, first_note, n_notes; } rowout_t;
static int cmp_rowout(const void *a, const void *b)
{
    const rowout_t *x = (const rowout_t *)a, *y = (const rowout_t *)b;
    return (x->row > y->row) - (x->row < y->row);
}

int ra_oracle_step(ra_oracle *o, const ra_event *ev, size_t n_ev,
                   ra_event *msgs, size_t msgs_cap, size_t *n_msgs,
                   ra_note *notes, size_t notes_cap, size_t *n_notes)
{
    if (!o || (!ev && n_ev)) return RA_E_INVAL;
    /* contract: a step() discards locals queued by the flood host model */
    if (o->loc_n) memset(o->loc_n, 0, o->n_rows);
    u8 *seen = (u8 *)calloc(o->n_rows, 1);
    /* validate grouping + capacity */
    for (size_t i = 0; i < n_ev;) {
        u32 row = ev[i].row;
        if (row >= o->n_rows || ev[i].type > RA_EV_CONSISTENT_QUERY || ev[i].type == RA_EV_NONE ||
            (ev[i].from_slot >= 15 && ev[i].from_slot != RA_NO_SLOT)) { free(seen); return RA_E_INVAL; }   /* sender slot: ra_engine.h */
        if (seen[row]) { free(seen); return RA_E_UNGROUPED; }
        seen[row] = 1;
        size_t j = i;
        while (j < n_ev && ev[j].row == row) j++;
        if (j - i > RA_LOCAL_CAP) { free(seen); return RA_E_CAPACITY; }
        i = j;
    }
    /* temp outputs in processing order, then ordered by row */
    size_t tm_cap = 0, tn_cap = 0, nro = 0;
    u32 routed = o->cfg.route_on_device;
    size_t touched = 0;
    /* rows to process: all rows with mail / pending (routed) plus rows in ev[] */
    u8 *todo = seen;   /* reuse: 1 = has caller events */
    for (u32 r = 0; r < o->n_rows; r++) {
        if (todo[r]) { touched++; continue; }
        int has = o->m[r].pipeline_pending;
        if (!has && routed)
            for (u32 s = 0; s < o->cfg.n_members && !has; s++)
                has = o->mbox_n[o->cur][(size_t)s * o->n_rows + r] != 0;
        if (has) { todo[r] = 2; touched++; }
    }
    tm_cap = touched * RA_MSG_CAP; tn_cap = touched * RA_NOTE_CAP;
    ra_event *tm = (ra_event *)malloc((tm_cap ? tm_cap : 1) * sizeof(ra_event));
    ra_note *tn = (ra_note *)malloc((tn_cap ? tn_cap : 1) * sizeof(ra_note));
    rowout_t *ro = (rowout_t *)malloc((touched ? touched : 1) * sizeof(rowout_t));
    size_t ntm = 0, ntn = 0;
    /* index of first caller event per row */
    size_t *first = (size_t *)malloc(((size_t)o->n_rows) * sizeof(size_t));
    for (size_t i = 0; i < n_ev; i++) if (i == 0 || ev[i - 1].row != ev[i].row) first[ev[i].row] = i;
    for (u32 r = 0; r < o->n_rows; r++) {
        if (!todo[r]) continue;
        member_t *m = &o->m[r];
        ctx_t c; ctx_begin(&c, o, m, &o->cnt, routed);
        if (!m->fatal) {
            process_row_prologue(&c);
            if (todo[r] == 1)
                for (size_t i = first[r]; i < n_ev && ev[i].row == r; i++) take_local(&c, &ev[i]);
        }
        publish_mbox_counts(&c);
        ctx_finish(&c);
        ro[nro].row = r; ro[nro].first_msg = (u32)ntm; ro[nro].n_msgs = c.n_msgs;
        ro[nro].first_note = (u32)ntn; ro[nro].n_notes = c.n_notes; nro++;
        memcpy(tm + ntm, c.msgs, c.n_msgs * sizeof(ra_event)); ntm += c.n_msgs;
        memcpy(tn + ntn, c.notes, c.n_notes * sizeof(ra_note)); ntn += c.n_notes;
    }
    if (routed) {
        /* rows that got nothing this step must still publish zero counts: the buffer we
           wrote into (cur^1) was cleared when it was last consumed, so nothing to do */
        o->cur ^= 1;
    }
    o->cnt.steps++;
    qsort(ro, nro, sizeof(rowout_t), cmp_rowout);
    int rc = RA_OK;
    if (ntm > msgs_cap || ntn > notes_cap) rc = RA_E_CAPACITY;
    else {
        size_t a = 0, b = 0;
        for (size_t i = 0; i < nro; i++) {
            memcpy(msgs + a, tm + ro[i].first_msg, ro[i].n_msgs * sizeof(ra_event)); a += ro[i].n_msgs;
            memcpy(notes + b, tn + ro[i].first_note, ro[i].n_notes * sizeof(ra_note)); b += ro[i].n_notes;
        }
        if (n_msgs) *n_msgs = a;
        if (n_notes) *n_notes = b;
    }
    free(tm); free(tn); free(ro); free(first); free(seen);
    return rc;
}

/* ------------------------------------------------------------------ */
/* flood: device transport + synthetic host model (DESIGN.md "flood")   */
/* ------------------------------------------------------------------ */
static u64 mix64(u64 x)
{   /* splitmix64 finaliser */
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

typedef struct {
    ra_oracle *o; u32 g0, g1; u32 n_steps, cmds, permille; u64 seed; ra_counters cnt;
    u64 step0; const struct flood_faults *ff;
} flood_arg_t;

/* host model for one row after its step: notes -> next step's local events */
static void host_model(ra_oracle *o, ctx_t *c, u64 step, u32 cmds, u32 permille, u64 seed)
{
    member_t *m = c->m;
    u32 row = m->row, G = o->cfg.n_groups, g = row % G;
    u64 gg = g, grow = row;                       /* ids the model hashes */
    if (o->s_stride) { gg = (u64)o->s_offset + (u64)g * o->s_stride; grow = (u64)m->self_slot * o->s_total + gg; }
    ra_event *loc = o->loc; u8 *ln = &o->loc_n[row];
    u32 k = 0;
    /* the last two WAL_APPEND notes become WRITTEN events */
    int w[2] = { -1, -1 };
    for (u32 i = 0; i < c->n_notes; i++)
        if (c->notes[i].type == RA_NOTE_WAL_APPEND) { w[0] = w[1]; w[1] = (int)i; }
    if (c->ff && c->ff->withhold && w[1] >= 0 &&           /* a lagging fsync: no notification this step */
        (u32)(mix64(seed ^ (step * 0xA0761D6478BD642Full) ^ (grow * 0xE7037ED1A0B428DBull)) >> 32) % 1000u < c->ff->withhold)
        w[0] = w[1] = -1;
    for (int j = 0; j < 2; j++) {
        if (w[j] < 0) continue;
        ra_event e; memset(&e, 0, sizeof e);
        e.row = row; e.type = RA_EV_WRITTEN; e.from_slot = RA_NO_SLOT;
        e.term = c->notes[w[j]].c; e.a = c->notes[w[j]].a; e.b = c->notes[w[j]].b;
        loc[(size_t)k * o->n_rows + row] = e; k++;
    }
    if (m->role == RA_LEADER && cmds > 0) {
        ra_event e; memset(&e, 0, sizeof e);
        e.row = row; e.type = RA_EV_COMMAND; e.from_slot = RA_NO_SLOT; e.n = cmds;
        loc[(size_t)k * o->n_rows + row] = e; k++;
    }
    /* election timer: steps without a leader message */
    int fire = 0;
    if (m->role == RA_LEADER || (c->status & RA_ST_LEADER_MSG)) m->idle = 0;
    else m->idle++;
    if (m->role != RA_LEADER) {
        u32 h = (u32)(mix64(seed ^ (step * 0x9E3779B97F4A7C15ull) ^ (gg * 0xD1B54A32D192ED03ull)) >> 32);
        if (permille && (h % 1000u) < permille && ((h / 1000u) % o->cfg.n_members) == m->self_slot) fire = 1;
        u32 h2 = (u32)(mix64(seed ^ (grow * 0xA24BAED4963EE407ull) ^ step) >> 32);
        if (m->idle >= 8 + (h2 & 7u)) fire = 1;
    }
    if (fire) {
        ra_event e; memset(&e, 0, sizeof e);
        e.row = row; e.type = RA_EV_ELECTION_TIMEOUT; e.from_slot = RA_NO_SLOT;
        loc[(size_t)k * o->n_rows + row] = e; k++;
        m->idle = 0;
    }
    *ln = (u8)k;
}

/* checker for big runs: this oracle's group g plays global group offset + g * stride of a flood over
   total_groups groups (groups are independent; the host model is the only thing keyed by their ids) */
int ra_oracle_set_sample(ra_oracle *o, uint32_t stride, uint32_t offset, uint32_t total_groups)
{
    if (!o || !stride || (uint64_t)offset + (uint64_t)(o->cfg.n_groups - 1) * stride >= total_groups) return RA_E_INVAL;
    o->s_stride = stride; o->s_offset = offset; o->s_total = total_groups;
    return RA_OK;
}

static void flood_groups(ra_oracle *o, u32 g0, u32 g1, u32 n_steps, u32 cmds, u32 permille,
                         u64 seed, u64 step0, ra_counters *cnt, const struct flood_faults *ff)
{
    u32 M = o->cfg.n_members, G = o->cfg.n_groups;
    /* groups are independent: a shard can run all its steps back to back.  `cur` is
       global, so each shard tracks its own parity starting from o->cur */
    int cur0 = o->cur;
    for (u32 t = 0; t < n_steps; t++) {
        int cur = cur0 ^ (int)(t & 1);
        for (u32 s = 0; s < M; s++) {
            for (u32 g = g0; g < g1; g++) {
                u32 row = s * G + g;
                member_t *m = &o->m[row];
                ctx_t c; ctx_begin(&c, o, m, cnt, 1);
                /* process_row_prologue/publish use o->cur: emulate with a local copy */
                ra_oracle view = *o; view.cur = cur; c.o = &view;
                c.ff = ff; c.ff_seed = seed; c.ff_step = step0 + t;
                if (!m->fatal) {
                    process_row_prologue(&c);
                    u32 nl = o->loc_n[row];
                    for (u32 k = 0; k < nl; k++) {
                        ra_event e = o->loc[(size_t)k * o->n_rows + row];
                        take_local(&c, &e);
                    }
                }
                o->loc_n[row] = 0;
                publish_mbox_counts(&c);
                ctx_finish(&c);
                c.o = o;
                if (!m->fatal) host_model(o, &c, step0 + t, cmds, permille, seed);
            }
        }
    }
}

static void *flood_thread(void *p)
{
    flood_arg_t *a = (flood_arg_t *)p;
    flood_groups(a->o, a->g0, a->g1, a->n_steps, a->cmds, a->permille, a->seed, a->step0, &a->cnt, a->ff);
    return NULL;
}

int ra_oracle_flood(ra_oracle *o, uint32_t n_steps, uint32_t cmds_per_step,
                    uint32_t election_permille, uint64_t seed, uint32_t threads)
{ return ra_oracle_flood_faults(o, n_steps, cmds_per_step, election_permille, seed, threads, NULL); }

int ra_oracle_flood_faults(ra_oracle *o, uint32_t n_steps, uint32_t cmds_per_step, uint32_t election_permille,
                           uint64_t seed, uint32_t threads, const ra_flood_faults *faults)
{
    if (!o || !o->cfg.route_on_device) return RA_E_INVAL;
    if (faults && faults->partition_permille && !faults->partition_steps) return RA_E_INVAL;
    struct flood_faults ffv, *ff = NULL;
    if (faults) { ffv.drop = faults->drop_permille; ffv.withhold = faults->withhold_permille;
                  ffv.part = faults->partition_permille; ffv.part_len = faults->partition_steps; ff = &ffv; }
    if (threads < 1) threads = 1;
    if (threads > o->cfg.n_groups) threads = o->cfg.n_groups;
    flood_arg_t *args = (flood_arg_t *)calloc(threads, sizeof *args);
    pthread_t *th = (pthread_t *)calloc(threads, sizeof *th);
    u32 G = o->cfg.n_groups;
    for (u32 i = 0; i < threads; i++) {
        args[i].o = o; args[i].g0 = (u32)((u64)G * i / threads); args[i].g1 = (u32)((u64)G * (i + 1) / threads);
        args[i].n_steps = n_steps; args[i].cmds = cmds_per_step; args[i].permille = election_permille;
        args[i].seed = seed; args[i].step0 = o->step_no; args[i].ff = ff;
        if (threads == 1) flood_thread(&args[i]);
        else pthread_create(&th[i], NULL, flood_thread, &args[i]);
    }
    for (u32 i = 0; i < threads; i++) {
        if (threads > 1) pthread_join(th[i], NULL);
        o->cnt.events += args[i].cnt.events; o->cnt.commits += args[i].cnt.commits;
        o->cnt.applied += args[i].cnt.applied; o->cnt.msgs_out += args[i].cnt.msgs_out;
        o->cnt.msgs_dropped += args[i].cnt.msgs_dropped;
        o->cnt.elections_won += args[i].cnt.elections_won;
        o->cnt.fatal_rows += args[i].cnt.fatal_rows;
        o->cnt.aer_received_follower += args[i].cnt.aer_received_follower;
        o->cnt.aer_received_follower_empty += args[i].cnt.aer_received_follower_empty;
        o->cnt.aer_replies_success += args[i].cnt.aer_replies_success;
        o->cnt.aer_replies_failed += args[i].cnt.aer_replies_failed;
        o->cnt.elections += args[i].cnt.elections;
        o->cnt.pre_vote_elections += args[i].cnt.pre_vote_elections;
        o->cnt.term_and_voted_for_updates += args[i].cnt.term_and_voted_for_updates;
    }
    o->cur ^= (int)(n_steps & 1);
    o->step_no += n_steps;
    o->cnt.steps += n_steps;
    free(args); free(th);
    return RA_OK;
}

/* ra_engine_step_host: the same step for a batch of 32-byte host-origin events */
int ra_oracle_step_host(ra_oracle *o, const ra_host_event *ev, size_t n_ev,
                        ra_event *msgs, size_t msgs_cap, size_t *n_msgs,
                        ra_note *notes, size_t notes_cap, size_t *n_notes)
{
    if (!o || (!ev && n_ev)) return RA_E_INVAL;
    ra_event *w = (ra_event *)calloc(n_ev ? n_ev : 1, sizeof(ra_event));
    if (!w) return RA_E_NOMEM;
    for (size_t i = 0; i < n_ev; i++) {
        const u8 t = ev[i].type;
        if (!(t == RA_EV_WRITTEN || t == RA_EV_COMMAND || t == RA_EV_ELECTION_TIMEOUT || t == RA_EV_AWAIT_COND_TIMEOUT ||
              t == RA_EV_PIPELINE_RPCS || t == RA_EV_TICK || t == RA_EV_CONSISTENT_QUERY)) { free(w); return RA_E_INVAL; }
        w[i].row = ev[i].row; w[i].type = t; w[i].from_slot = RA_NO_SLOT; w[i].flags = ev[i].flags; w[i].n = ev[i].n;
        w[i].term = ev[i].term; w[i].a = ev[i].a; w[i].b = ev[i].b;
    }
    int rc = ra_oracle_step(o, w, n_ev, msgs, msgs_cap, n_msgs, notes, notes_cap, n_notes);
    free(w);
    return rc;
}

int ra_oracle_counters(ra_oracle *o, ra_counters *out)
{
    if (!o || !out) return RA_E_INVAL;
    *out = o->cnt;
    return RA_OK;
}
