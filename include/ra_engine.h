/*
 * ra_engine.h -- C ABI of the H100 batched multi-Raft engine.
 *
 * Drop-in boundary: the call from ra_server_proc into the pure Raft core,
 *   ra_server:handle_leader(Msg, State)            src/ra_server_proc.erl:1354
 *   ra_server:RaftState(Msg, State)                src/ra_server_proc.erl:1383
 * both returning {NextRaftState, NewState, Effects} (src/ra_server.erl:520-521).
 * The reference has no FFI for this path (it is 100 % Erlang); the entry points
 * below are what a dirty-NIF shim binds (see INTEGRATION.md).  Every struct is
 * plain-old-data, little endian, no pointers inside, no torch types.
 *
 * Vocabulary follows the reference: member, peer, term, index, commit_index,
 * last_applied, last_written, append_entries_rpc (AER), pre_vote, ...
 *
 * A "row" is one Raft member (one ra_server_state()).  Members of group g are
 * rows  slot * n_groups + g  for slot in [0, n_members): slot-major, so that
 * the same slot of consecutive groups is contiguous in every HBM column.
 */
#ifndef RA_ENGINE_H
#define RA_ENGINE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RA_MAX_MEMBERS   8      /* members per group (slots 0..7)                    */
#define RA_MAX_RUNS      8      /* term runs kept per member log view                */
#define RA_NO_SLOT       0xFFu  /* 'undefined' for leader_id / voted_for             */
#define RA_UNDEF_TERM    UINT64_MAX /* fetch_term -> undefined                         */
#define RA_MBOX_DEPTH    4      /* per (src,dst) messages per step in routed mode    */
#define RA_LOCAL_CAP     4      /* host ("local") events per row per step            */
#define RA_MSG_CAP       16     /* outgoing RPC records per row per step             */
#define RA_NOTE_CAP      16     /* host notes per row per step (cfg.note_cap may lower it) */
#define RA_NOTE_RESERVE  4      /* a row takes its next event of a step only while at least this many
                                   note slots (+ the one kept for STATUS) are free, so that no event's
                                   notes are ever cut off half-way: see "note budget" below  */

/* ra_state(), src/ra_server.erl:116-119 (the five states on the hot path) */
enum ra_role {
    RA_FOLLOWER        = 0,
    RA_CANDIDATE       = 1,
    RA_PRE_VOTE        = 2,
    RA_LEADER          = 3,
    RA_AWAIT_CONDITION = 4
};

/* ra_membership(), src/ra.hrl:58 */
enum ra_membership {
    RA_VOTER      = 0,
    RA_PROMOTABLE = 1,
    RA_NON_VOTER  = 2,
    RA_UNKNOWN    = 3
};

/* ra_peer_status(), src/ra.hrl:52-56 (pids/attempt counts stay on the host) */
enum ra_peer_status {
    RA_PEER_NORMAL           = 0,
    RA_PEER_SENDING_SNAPSHOT = 1,
    RA_PEER_SNAPSHOT_BACKOFF = 2,
    RA_PEER_SUSPENDED        = 3,
    RA_PEER_DISCONNECTED     = 4
};

/* ra_msg(), src/ra_server.erl:144-164 -- the subset evaluated on the GPU */
enum ra_event_type {
    RA_EV_NONE              = 0,
    RA_EV_AER               = 1,  /* #append_entries_rpc{}      src/ra.hrl:122-128 */
    RA_EV_AER_REPLY         = 2,  /* {Peer,#append_entries_reply{}}      :130-141 */
    RA_EV_REQUEST_VOTE      = 3,  /* #request_vote_rpc{}                  :144-148 */
    RA_EV_REQUEST_VOTE_RES  = 4,  /* #request_vote_result{}               :151-153 */
    RA_EV_PRE_VOTE          = 5,  /* #pre_vote_rpc{}                      :156-164 */
    RA_EV_PRE_VOTE_RES      = 6,  /* #pre_vote_result{}                   :166-169 */
    RA_EV_WRITTEN           = 7,  /* {ra_log_event,{written,Term,Seq}}  ra_log.erl:73 */
    RA_EV_COMMAND           = 8,  /* {command,_} / {commands,_} ra_server.erl:644-729 */
    RA_EV_ELECTION_TIMEOUT  = 9,  /* election_timeout                              */
    RA_EV_AWAIT_COND_TIMEOUT= 10, /* await_condition_timeout                       */
    RA_EV_PIPELINE_RPCS     = 11, /* pipeline_rpcs            ra_server.erl:784-792 */
    RA_EV_TICK              = 12, /* leader tick -> make_rpcs ra_server_proc.erl:610 */
    /* consistent queries (SURVEY 8f-3): the heartbeat round of ra_server.erl:846-918, :3700-3825 */
    RA_EV_HEARTBEAT_RPC     = 13, /* #heartbeat_rpc{}   from_slot=leader term a=query_index          */
    RA_EV_HEARTBEAT_REPLY   = 14, /* {Peer,#heartbeat_reply{}}  from_slot=peer term a=query_index    */
    RA_EV_CONSISTENT_QUERY  = 15  /* {consistent_query|consistent_aux,_,_} handed to the leader; the
                                     host holds the query refs and submits one only while cluster
                                     changes are permitted (it keeps `pending_consistent_queries`)  */
};

/* ra_event.flags */
#define RA_EVF_NOOP        0x01u /* COMMAND: entry is {noop,_,_} (forces pipelining, :674-679) */
#define RA_EVF_NEXT_EVENT  0x02u /* out only, pure mode: {next_event, Msg} addressed to self   */
#define RA_EVF_INFO        0x08u /* next_event type was `info` (pipeline_rpcs)                 */

/*
 * One 64-byte wire record.  Used for (a) events fed to the engine and (b) RPC
 * records the engine emits (they are already addressed: `row` = destination).
 *
 *  type            from_slot   term      a               b              c              d            e
 *  AER             leader      rpc term  prev_log_index  prev_log_term  leader_commit  entry term   term of the entries after the
 *                                                                                                    first n1 (used when n1 != 0)
 *                  n = number of entries (prev+1 .. prev+n); n1 = 0: all have term d, else the first
 *                  n1 have term d and the other n-n1 have term e (an AER spans <= 2 term runs)
 *  AER_REPLY       replier     term      next_index      last_index     last_term      success(0/1)
 *  REQUEST_VOTE    candidate   term      last_log_index  last_log_term
 *  REQUEST_VOTE_RES voter      term      -               -              -              granted(0/1)
 *  PRE_VOTE        candidate   term      last_log_index  last_log_term  token          version | machine_version<<32
 *  PRE_VOTE_RES    voter       term      -               -              token          granted(0/1)
 *  WRITTEN         -           term      from            to                                        (Seq = [{from,to}])
 *  COMMAND         -           -         -               -              -              -            n = number of commands
 *  HEARTBEAT_RPC   leader      term      query_index
 *  HEARTBEAT_REPLY replier     term      query_index
 *  CONSISTENT_QUERY -
 */
typedef struct ra_event {
    uint32_t row;        /* destination member row                                  */
    uint8_t  type;       /* enum ra_event_type                                      */
    uint8_t  from_slot;  /* sender's slot in the group, RA_NO_SLOT for host events  */
    uint8_t  flags;      /* RA_EVF_*                                                */
    uint8_t  _pad;
    uint16_t n;          /* entry / command count                                   */
    uint16_t n1;         /* AER: entries in the first term run (0 = all)            */
    uint32_t seq;        /* out records: k-th record of its row in this step        */
    uint64_t term;
    uint64_t a, b, c, d;
    uint64_t e;
} ra_event;

/* Host notes: what ra_server_proc must do that the engine cannot (32 bytes). */
enum ra_note_type {
    RA_NOTE_NONE       = 0,
    RA_NOTE_WAL_APPEND = 1, /* a=from b=to c=term of `to`: entries now in the log view;
                               host writes payloads (ra_log:append / ra_log:write)        */
    RA_NOTE_TRUNCATE   = 2, /* a=new last index b=its term   (ra_log:set_last_index)      */
    RA_NOTE_COMMIT     = 3, /* a=old commit_index b=new      ({aux,eval}, :3611-3614)     */
    RA_NOTE_APPLY      = 4, /* a=first b=last index to run through ra_machine:apply/3     */
    RA_NOTE_STATUS     = 5, /* end-of-step summary: aux=flags, a=term, b=voted_for|leader<<8|
                               role_old<<16|role_new<<24, c=detail.  When the only flag is
                               RA_ST_LEADER_MSG and the row has another note in this step, there is
                               no STATUS note: the flags are the aux of the row's LAST note       */
    RA_NOTE_SEND_SNAPSHOT = 6, /* a=peer slot b=snapshot index  ({send_snapshot,..} :2395) */
    RA_NOTE_NOT_LEADER = 7, /* COMMAND / CONSISTENT_QUERY reached a non-leader: a=n commands b=leader slot */
    RA_NOTE_QUERY_INDEX = 8,  /* the query just submitted waits for heartbeats: a=its query_index
                                 b=commit_index it must read at (queries_waiting_heartbeats, :3722-3739) */
    RA_NOTE_QUERY_AGREED = 9, /* a=query_index a quorum has confirmed: every waiting query <= a is
                                 applied by the host (heartbeat_rpc_quorum/3, :3766-3784)              */
    RA_NOTE_QUERY_APPLY = 10, /* no peers: apply the query just submitted right away (:3729-3731)      */
    RA_NOTE_CANCEL_SNAPSHOT_RETRY = 11 /* slot=a=peer: {cancel_snapshot_retry_timer, Peer}: make_all_rpcs/1
                                 (:2337-2350) also reaches out to a peer in snapshot_backoff          */
};

/* RA_NOTE_STATUS aux flags */
#define RA_ST_TERM_VOTE_CHANGED   0x0001u /* update_term_and_voted_for persisted (:3014-3031)    */
#define RA_ST_ROLE_CHANGED        0x0002u
#define RA_ST_LEADER_MSG          0x0004u /* {record_leader_msg,_} (:1280)                        */
#define RA_ST_START_ELECTION_TMO  0x0008u /* start_election_timeout effect (:2934,2942)           */
#define RA_ST_MSG_DROPPED         0x0010u /* an outgoing record did not fit (transport full)      */
#define RA_ST_PIPELINE_PENDING    0x0020u /* pipeline_rpcs continues next step                    */
#define RA_ST_FATAL               0x0040u /* c = enum ra_fatal; the reference would exit/crash    */
#define RA_ST_CMD_POSTPONED       0x0080u /* COMMAND while in await_condition (proc postpones)    */
#define RA_ST_BECAME_LEADER       0x0100u
#define RA_ST_NOTE_OVERFLOW       0x0200u /* note budget: the row stopped taking events for this step.  Mailbox
                                             records it had not reached are dropped (and counted, like a full
                                             transport); the host events it had not reached were NOT consumed:
                                             STATUS.c bits 8..15 = how many (the LAST ones of the row's run in
                                             ev[]) -- submit them again in the next call                        */

enum ra_fatal {
    RA_FATAL_NONE = 0,
    RA_FATAL_LEADER_SAW_AER_SAME_TERM = 1, /* exit(leader_saw_append_entries_rpc_in_same_term) :840 */
    RA_FATAL_WRITE_INTEGRITY = 2,          /* ra_log:write/2 {error,{integrity_error,_}}  :1369    */
    RA_FATAL_SET_LAST_INDEX_NOT_FOUND = 3, /* {ok,L} = ra_log:set_last_index(..) badmatch :1301    */
    RA_FATAL_ASSERT = 4,                   /* a ?assert / ?assertNot in the reference failed       */
    RA_FATAL_NO_SNAPSHOT = 5,              /* make_rpc_effect: prev entry and snapshot both absent :2378 */
    RA_FATAL_LEADER_SAW_HEARTBEAT_SAME_TERM = 6, /* exit(leader_saw_heartbeat_rpc_in_same_term) :894 */
    RA_FATAL_NOTE_OVERFLOW = 7             /* one event produced more notes than the budget reserves (only a burst
                                              of SEND_SNAPSHOT / CANCEL_SNAPSHOT_RETRY notes can): nothing is lost
                                              silently -- the row stops like a crashed server and is reloaded    */
};

typedef struct ra_note {
    uint32_t row;
    uint8_t  type;     /* enum ra_note_type */
    uint8_t  slot;
    uint16_t aux;
    uint64_t a, b, c;
} ra_note;

/* One peer entry of ra_cluster() / ra_peer_state(), src/ra.hrl:63-75 */
typedef struct ra_peer_init {
    uint64_t next_index;          /* new_peer/0: 1   src/ra_server.erl:2963-2968 */
    uint64_t match_index;         /* 0 */
    uint64_t commit_index_sent;   /* 0 */
    uint8_t  status;              /* enum ra_peer_status */
    uint8_t  voter;               /* 1 unless voter_status.membership =/= voter */
    uint8_t  _pad[6];
} ra_peer_init;

/*
 * Everything ra_server:init/1 (src/ra_server.erl:434-457) + the log facade hold
 * for one member, as far as the hot path reads it.  Used to load rows and to
 * read them back for a parity diff.
 */
typedef struct ra_row_state {
    uint32_t row;
    uint8_t  role;                /* enum ra_role */
    uint8_t  self_slot;
    uint8_t  n_members;
    uint8_t  leader_slot;         /* RA_NO_SLOT = undefined */
    uint8_t  voted_for;           /* RA_NO_SLOT = undefined */
    uint8_t  membership;          /* enum ra_membership of this member */
    uint8_t  condition;           /* 0 none, 1 catch-up(missing), 2 catch-up(term_mismatch) */
    uint8_t  has_snapshot;
    uint32_t votes;
    uint32_t machine_version;             /* #cfg.machine_version            */
    uint32_t effective_machine_version;   /* #cfg.effective_machine_version  */
    uint32_t n_runs;
    uint32_t flags;               /* bit0: pipeline_rpcs pending, bit1: cond reply valid */
    uint64_t current_term;
    uint64_t commit_index;
    uint64_t last_applied;
    uint64_t pre_vote_token;
    uint64_t token_counter;
    /* log view (ra_log facade): range [first_index,last_index] */
    uint64_t first_index;
    uint64_t last_index;
    uint64_t last_term;
    uint64_t last_written_index;
    uint64_t last_written_term;
    uint64_t snapshot_index;
    uint64_t snapshot_term;
    /* index->term knowledge as runs: entries run_start[i] .. (run_start[i+1]-1 | last_index)
       have term run_term[i]; runs are ascending in start index.                        */
    uint64_t run_start[RA_MAX_RUNS];
    uint64_t run_term[RA_MAX_RUNS];
    /* await_condition timeout effect: the reply to repeat (src/ra_server.erl:1383-1386) */
    uint64_t cond_reply_term, cond_reply_next_index, cond_reply_last_index, cond_reply_last_term;
    ra_peer_init peers[RA_MAX_MEMBERS];   /* indexed by slot; entry self_slot mirrors the
                                             reference keeping itself in the cluster map  */
} ra_row_state;

typedef struct ra_engine_cfg {
    uint32_t n_groups;            /* rows = n_groups * n_members                          */
    uint32_t n_members;           /* 1..RA_MAX_MEMBERS                                    */
    uint32_t max_pipeline_count;  /* ?DEFAULT_MAX_PIPELINE_COUNT 4096  src/ra_server.hrl:8 */
    uint32_t max_aer_batch;       /* ?AER_CHUNK_SIZE 128               src/ra_server.hrl:7 */
    int32_t  device;              /* CUDA device ordinal                                  */
    uint32_t route_on_device;     /* 1: RPC records for rows of this engine are delivered
                                     through HBM mailboxes (benchmark transport), never
                                     shown to the host.  0: every RPC record is returned.
                                     BENCHMARK / CLOSED-LOOP TESTS ONLY: a row's replies reach their
                                     destination in the same step that sets RA_ST_TERM_VOTE_CHANGED,
                                     before the host could persist term / voted_for
                                     (ra_server.erl:3024-3025); a real integration uses 0, persists,
                                     then sends.                                                    */
    uint32_t pure;                /* 1: do not chase {next_event,_}; return it as a record
                                     (the shape ra_server_SUITE asserts on)               */
    uint32_t n_shards;            /* 0 or 1: every member of a group lives in this engine.  N > 1 (needs
                                     route_on_device): member (group g, slot s) lives in the engine with
                                     shard == (g + s) mod N, at local group index g div N; n_groups is then
                                     the LOCAL group count per slot.  RPC records for other shards go to the
                                     outbox (ra_engine_set_outbox) and come back through ra_engine_deliver */
    uint32_t shard;
    uint32_t note_cap;            /* 0 = RA_NOTE_CAP; else notes per row per step, RA_NOTE_RESERVE + 2 .. RA_NOTE_CAP
                                     (a smaller value only makes the note budget bite earlier: tests)      */
} ra_engine_cfg;

typedef struct ra_engine ra_engine;

typedef struct ra_counters {
    uint64_t events;              /* events evaluated                                     */
    uint64_t commits;             /* sum of commit_index advances on leaders (the metric) */
    uint64_t applied;             /* sum of last_applied advances                         */
    uint64_t msgs_out;            /* RPC records emitted                                  */
    uint64_t msgs_dropped;        /* RPC records that found the transport full            */
    uint64_t elections_won;
    uint64_t fatal_rows;
    uint64_t steps;
    /* the reference's own counters of this path (src/ra.hrl:324-343), summed over all members */
    uint64_t aer_received_follower;        /* ?C_RA_SRV_AER_RECEIVED_FOLLOWER        ra_server.erl:1278,1418 */
    uint64_t aer_received_follower_empty;  /* ?C_RA_SRV_AER_RECEIVED_FOLLOWER_EMPTY  :1290 */
    uint64_t aer_replies_success;          /* ?C_RA_SRV_AER_REPLIES_SUCCESS          :528  */
    uint64_t aer_replies_failed;           /* ?C_RA_SRV_AER_REPLIES_FAILED           :590  */
    uint64_t elections;                    /* ?C_RA_SRV_ELECTIONS                    :2856 */
    uint64_t pre_vote_elections;           /* ?C_RA_SRV_PRE_VOTE_ELECTIONS           :2878 */
    uint64_t term_and_voted_for_updates;   /* ?C_RA_SRV_TERM_AND_VOTED_FOR_UPDATES   :3026 */
} ra_counters;

enum ra_status {
    RA_OK = 0,
    RA_E_INVAL = -1,      /* bad argument                                   */
    RA_E_NOMEM = -2,
    RA_E_CUDA = -3,       /* CUDA runtime error, see ra_engine_strerror     */
    RA_E_UNGROUPED = -4,  /* events of one row are not adjacent in the batch */
    RA_E_CAPACITY = -5,   /* more than RA_LOCAL_CAP events for one row, or out buffers too small */
    RA_E_NODEVICE = -6,
    RA_E_BUSY = -7        /* submit/collect: no free slot, or a submitted batch is still to be collected */
};

/* Lifecycle.  The engine owns the HBM Struct-of-Arrays; callers own all host buffers and
   the engine never keeps a host pointer past a call.  One engine per GPU; calls on one
   engine must be serialised (as gen_statem serialises one member's mailbox).
   Index width: every index and term of this ABI is 64 bits wide and is evaluated as such.  Internally the hot
   kernel keeps a member's values in 32-bit registers while ALL of them are below 2^30 and hands a member (or a
   record) that has outgrown that to the 64-bit kernels -- results are bit-identical either way.  Environment, read
   at create time, performance only: RA_STEP_WIDE=1 never uses the 32-bit hot kernel, RA_STEP_WIDE=0 always does,
   unset = a bulk ra_engine_load_rows (>= half the rows) decides by what it loads.               */
int  ra_engine_create(const ra_engine_cfg* cfg, ra_engine** out);
void ra_engine_destroy(ra_engine* e);
int  ra_engine_get_cfg(ra_engine* e, ra_engine_cfg* out);

/* = ra_server:init/1 values (src/ra_server.erl:434-457) + log tail, per row. */
int  ra_engine_load_rows(ra_engine* e, const ra_row_state* rows, size_t n);
/* What load_rows requires of the log view of a row (RA_E_INVAL otherwise): n_runs <= RA_MAX_RUNS; the log
 * is empty (first_index > last_index, n_runs = 0) or its runs start at first_index, ascend strictly, stay
 * inside [first_index, last_index], carry non-decreasing terms and end in last_term; slots < RA_MAX_MEMBERS. */
static inline int ra_row_state_valid(const ra_row_state* s)
{
    if (s->n_runs > RA_MAX_RUNS || s->n_members < 1 || s->n_members > RA_MAX_MEMBERS || s->self_slot >= s->n_members) return 0;
    if (s->role > RA_AWAIT_CONDITION || s->membership > RA_UNKNOWN || s->condition > 2) return 0;
    /* leader_id / voted_for may name a server outside the cluster map (the reference keeps whatever id it was told):
       any slot below 15 or RA_NO_SLOT is representable */
    if ((s->leader_slot != RA_NO_SLOT && s->leader_slot >= 15) || (s->voted_for != RA_NO_SLOT && s->voted_for >= 15)) return 0;
    for (uint32_t p = 0; p < RA_MAX_MEMBERS; p++) if (s->peers[p].status > RA_PEER_DISCONNECTED) return 0;
    if (s->n_runs == 0) return s->first_index > s->last_index;
    if (s->first_index > s->last_index || s->run_start[0] != s->first_index) return 0;
    for (uint32_t k = 1; k < s->n_runs; k++)
        if (s->run_start[k] <= s->run_start[k - 1] || s->run_term[k] < s->run_term[k - 1]) return 0;
    return s->run_start[s->n_runs - 1] <= s->last_index && s->run_term[s->n_runs - 1] == s->last_term;
}

/* Convenience: every row := ra_server_SUITE:empty_state/2 (:4022-4032), current_term 0. */
int  ra_engine_reset_empty(ra_engine* e);
/* For the parity diff. `rows[i].row` selects the row; the rest is filled in. */
int  ra_engine_read_rows(ra_engine* e, ra_row_state* rows, size_t n);

/* Consistent-query state of a member (kept apart from ra_row_state): its own query_index
 * (ra_server_state(), :96), every peer's (ra_peer_state(), ra.hrl:63-75) and the highest index the
 * host has been told a quorum agreed on.  load/read like the rows; zero after reset / load_rows. */
typedef struct ra_query_state {
    uint32_t row, _pad;
    uint64_t query_index;
    uint64_t agreed_index;
    uint64_t peer_query_index[RA_MAX_MEMBERS];
} ra_query_state;
int  ra_engine_load_query_state(ra_engine* e, const ra_query_state* q, size_t n);
int  ra_engine_read_query_state(ra_engine* e, ra_query_state* q, size_t n);

/*
 * Evaluate one batch.  ev[0..n_ev): events for one row must be adjacent and are applied
 * in array order (= mailbox order); at most RA_LOCAL_CAP per row per call.  In
 * route_on_device mode mailbox records delivered by the previous step are evaluated first
 * (by sender slot, then send order), then ev[].  Outputs: RPC records (already addressed)
 * and host notes, each ordered by (row, seq).  Returns RA_OK or a negative ra_status.
 */
int  ra_engine_step(ra_engine* e,
                    const ra_event* ev, size_t n_ev,
                    ra_event* msgs, size_t msgs_cap, size_t* n_msgs,
                    ra_note*  notes, size_t notes_cap, size_t* n_notes);

/*
 * Capacity.  A row emits at most RA_MSG_CAP records and RA_NOTE_CAP notes per step, and rows WITHOUT an
 * event in the batch can emit too (a deferred pipeline pass, mailbox records in route_on_device mode), so
 * n_ev * CAP is not a bound -- rows * CAP is.  A call whose outputs exceed msgs_cap / notes_cap returns
 * RA_E_CAPACITY with *n_msgs / *n_notes = the sizes needed; the step HAS been evaluated and nothing is lost:
 * the outputs stay in the engine until ra_engine_fetch_output takes them (no other step call is accepted
 * before that).  RA_E_CAPACITY for more than RA_LOCAL_CAP events of one row, RA_E_UNGROUPED and RA_E_INVAL
 * (bad row / type) reject the whole batch: no row has changed.
 */
int  ra_engine_pending_output(ra_engine* e, size_t* n_msgs, size_t* n_notes);
int  ra_engine_fetch_output(ra_engine* e, ra_event* msgs, size_t msgs_cap, size_t* n_msgs,
                            ra_note* notes, size_t notes_cap, size_t* n_notes);

/*
 * Benchmark transport + synthetic host, all on the device (no host copies):
 * one step = [deliver mailboxes] + raft_step + [host model: every WAL_APPEND note becomes
 * the matching WRITTEN event of the next step; every leader gets COMMAND(n=cmds_per_step)].
 * election_permille: per step, that fraction (x/1000) of groups get election_timeout on a
 * follower chosen by hash(seed, step, group).  Returns after the work is enqueued on the
 * engine's stream; ra_engine_sync() waits for it.
 */
int  ra_engine_flood(ra_engine* e, uint32_t n_steps, uint32_t cmds_per_step,
                     uint32_t election_permille, uint64_t seed);
/*
 * The same flood with fault injection (BASELINE.json configs[4]: follower lag / log-mismatch): all deterministic,
 * keyed by (seed, step, GLOBAL group / row ids), so the CPU oracle and a sharded run reproduce them exactly.
 *   drop_permille       an AppendEntries record evaluated at step t by row r from sender s is lost iff
 *                       hi32(mix64(seed ^ t*K1 ^ r*K2 ^ (s+1)<<56)) mod 1000 < drop_permille  (-> `missing` ->
 *                       await_condition -> failure reply -> next_index back-off)
 *   withhold_permille   the WRITTEN events for a row's WAL_APPEND notes of step t are not produced (a lagging
 *                       fsync: a later notification covers the range) iff hash(seed, t, r) mod 1000 < it
 *   partition_permille  in every window of partition_steps steps, a group has one member cut off with that
 *                       probability (chosen by hash(seed, window, group)): it evaluates no mailbox record and
 *                       nobody evaluates a record from it.  When it is the leader the others elect a new one and
 *                       the old leader later rejoins with an unreplicated tail (term-conflict / truncate path).
 * Lost records are counted in msgs_dropped.  All zero = ra_engine_flood.
 */
typedef struct ra_flood_faults {
    uint32_t drop_permille, withhold_permille, partition_permille, partition_steps;
} ra_flood_faults;
int  ra_engine_flood_faults(ra_engine* e, uint32_t n_steps, uint32_t cmds_per_step, uint32_t election_permille,
                            uint64_t seed, const ra_flood_faults* faults);
int  ra_engine_sync(ra_engine* e);
int  ra_engine_counters(ra_engine* e, ra_counters* out);     /* syncs */
/* diagnostics: out[role * 16 + event_type] = events that were not covered by a steady-state fast
   path and went through the general kernel (8 roles x 16 types = 128 counters) */
int  ra_engine_stall_histogram(ra_engine* e, uint64_t* out128);
/* elapsed device time (ms) of the raft_step kernel over the last flood call, CUDA events
   on the engine's stream, and its launch count */
int  ra_engine_last_kernel_ms(ra_engine* e, float* ms, uint32_t* launches);

/*
 * Cross-shard transport (n_shards > 1).  The caller owns the exchange (NCCL all-to-all in
 * ra_b200/sharded.py): `outbox` is n_shards buckets of `cap` 64-byte records, bucket d holds the
 * records for shard d of the current step, counts[d] their number (both DEVICE pointers, reset by
 * the engine before every step).  ra_engine_deliver scatters what other shards sent into this
 * engine's mailboxes for the next step: bucket b = records from shard b, counts[b] of them.
 * ra_engine_set_stream makes the engine enqueue on the caller's CUDA stream (e.g. the one NCCL
 * collectives are ordered on).
 */
int  ra_engine_set_stream(ra_engine* e, void* cuda_stream);
int  ra_engine_set_outbox(ra_engine* e, void* outbox, uint32_t* counts, uint32_t cap);
int  ra_engine_deliver(ra_engine* e, const void* inbox, const uint32_t* counts, uint32_t cap);

/*
 * Peer transport (n_shards <= 8, GPUs of one NVLink/NVSwitch domain): instead of bucket +
 * all-to-all + deliver, every shard maps the mailbox buffers of the others and the step kernels
 * store each RPC record straight into the destination GPU's mailbox plane over NVLink -- compute
 * and transfer are one kernel.  The caller only has to keep the shards in lock step (one barrier
 * between steps).  ra_engine_peer_get returns this engine's buffers as device pointers (same
 * process) ; ra_engine_ipc_export / _import move them between processes as CUDA IPC handles.
 * ra_engine_peer_set(shard, ...) registers shard's buffers; once all n_shards are registered
 * (own shard included automatically) the kernels switch to peer stores.
 */
typedef struct ra_peer_ptrs { void* mbox[2]; void* mbox_cnt[2]; } ra_peer_ptrs;
typedef struct ra_ipc_handles { unsigned char h[4][64]; } ra_ipc_handles;
int  ra_engine_peer_get(ra_engine* e, ra_peer_ptrs* out);
int  ra_engine_peer_set(ra_engine* e, uint32_t shard, const ra_peer_ptrs* p);
int  ra_engine_ipc_export(ra_engine* e, ra_ipc_handles* out);
int  ra_engine_ipc_import(ra_engine* e, uint32_t shard, const ra_ipc_handles* h);
/* Peer transport, one shard per process: the step barrier as a kernel on the engine's stream (flag
 * words in every peer's HBM, release / acquire at system scope) instead of a collective.  All shards
 * must have the same number of rows; never use it with several shards on ONE stream. */
int  ra_engine_peer_barrier(ra_engine* e);
/* on != 0: ra_engine_flood ends every step with that barrier, so a multi-step flood of one shard per process
 * runs without the host between steps (one process per GPU only: see above) */
int  ra_engine_set_flood_barrier(ra_engine* e, int on);

/*
 * The same call for batches made only of events the HOST originates (written, command(s), timeouts, tick,
 * pipeline_rpcs, consistent_query): 32-byte records, half the host->device bytes of a step.  Same grouping
 * contract, same outputs; an RPC type in such a batch is RA_E_INVAL.
 */
typedef struct ra_host_event {
    uint32_t row;
    uint8_t  type;       /* enum ra_event_type, host-origin types only */
    uint8_t  flags;      /* RA_EVF_*                                   */
    uint16_t n;          /* COMMAND: number of commands                */
    uint64_t term, a, b; /* WRITTEN: term, from, to                    */
} ra_host_event;
int  ra_engine_step_host(ra_engine* e, const ra_host_event* ev, size_t n_ev,
                         ra_event* msgs, size_t msgs_cap, size_t* n_msgs,
                         ra_note* notes, size_t notes_cap, size_t* n_notes);

/*
 * Split-phase form of ra_engine_step[_host].  submit enqueues the whole call -- host->device copy of the
 * batch, the kernels, and the write-back of the outputs, which the last kernel stores straight into the
 * caller's buffers when they are pinned (ra_engine_alloc_host / ra_engine_register_host; into an internal
 * pinned staging area otherwise) -- and returns without waiting; collect waits for the OLDEST submitted call
 * and returns its status and output counts.  Up to two calls may be in flight per engine (the copy of batch
 * t+1 overlaps the kernels and the output of batch t); RA_E_BUSY beyond that.  The buffers of a submitted call
 * (ev, msgs, notes) belong to the engine until it is collected.  With several engines (disjoint sets of
 * groups) one host thread keeps all of them busy: submit to each, then collect each.
 * If a batch is rejected (ungrouped / capacity / bad row), collect returns the error, no row has changed, and
 * every call submitted behind it is rejected with the same status.
 */
int  ra_engine_submit(ra_engine* e, const ra_event* ev, size_t n_ev,
                      ra_event* msgs, size_t msgs_cap, ra_note* notes, size_t notes_cap);
int  ra_engine_submit_host(ra_engine* e, const ra_host_event* ev, size_t n_ev,
                           ra_event* msgs, size_t msgs_cap, ra_note* notes, size_t notes_cap);
/* the same batch handed over in pieces -- one per producer thread, each in its own (pinned) buffer -- which the engine
 * copies back to back: no host-side concatenation.  The grouping contract holds for the concatenation; a row's
 * events must not be split between two pieces.  At most 256 pieces. */
typedef struct ra_host_event_seg { const ra_host_event* ev; size_t n; } ra_host_event_seg;
int  ra_engine_submit_host_segs(ra_engine* e, const ra_host_event_seg* segs, size_t n_segs,
                                ra_event* msgs, size_t msgs_cap, ra_note* notes, size_t notes_cap);
int  ra_engine_collect(ra_engine* e, size_t* n_msgs, size_t* n_notes);
/*
 * Compact note stream.  With ra_engine_set_note_format(e, 1) the `notes` buffer of step / submit / fetch_output
 * receives 16-byte units instead of 32-byte ra_note records (notes_cap and *n_notes then count units / notes):
 *
 *   units[0 .. n_notes)                 one ra_note16 per note, ordered by (row, seq) like the notes
 *   units[n_notes .. n_notes + 2*n_ext) the extension area: n_ext entries of {a, b}, {c, 0}  (ra_engine_last_ext_count)
 *
 * A note {row, type, slot, aux, a, b, c} is ONE unit {row, type, n, aux, a} when slot = 0, 0 <= b - a < 256 (n = b - a)
 * and c is derivable: 0, or -- WAL_APPEND only, flagged RA_N16_SAME_TERM -- the c of this row's previous WAL_APPEND
 * note (the decoder keeps that per row, starting from 0 at reset / load / format switch; every WAL_APPEND note,
 * compact or not, updates it).  Any other note has RA_N16_EXT set: `n` is its slot, `a` the index of its extension
 * entry.  In the steady-state flood every note is compact: half the device->host bytes.  ra_notes16_expand is the
 * decoder (host code): it rebuilds the ra_note records.
 */
typedef struct ra_note16 {
    uint32_t row;
    uint8_t  type;       /* enum ra_note_type | RA_N16_EXT | RA_N16_SAME_TERM */
    uint8_t  n;          /* b - a, or the slot of an extended note            */
    uint16_t aux;
    uint64_t a;          /* a, or the extension index of an extended note     */
} ra_note16;
#define RA_N16_EXT        0x80u
#define RA_N16_SAME_TERM  0x40u
int    ra_engine_set_note_format(ra_engine* e, int compact);   /* only while no call is in flight */
size_t ra_engine_last_ext_count(ra_engine* e);                 /* n_ext of the call collected last */
/* units + extension area -> ra_note records; last_wal_c = the caller's per-row array (n_rows entries, zeroed at
   reset / load / format switch).  Returns the number of notes written (n_notes), or 0 if cap < n_notes. */
size_t ra_notes16_expand(const ra_note16* units, size_t n_notes, size_t n_ext, uint64_t* last_wal_c,
                         ra_note* out, size_t cap);

/* pin + map caller-owned host memory once (cudaHostRegister), e.g. a NIF's resource buffers */
int  ra_engine_register_host(void* p, size_t bytes);
int  ra_engine_unregister_host(void* p);


/*
 * Written-event source (SURVEY 8f-2): ra_log_wal:complete_batch/1 (src/ra_log_wal.erl:784-808) tells every
 * writer of a WAL batch {ra_log_event, {written, Term, Seq}} with Seq a ra_seq (src/ra_seq.erl: ascending
 * indexes and {From, To} ranges).  ra_wal_batch_to_events turns one batch -- an array of writers -- into the
 * grouped event array of ra_engine_step: one RA_EV_WRITTEN per range, ranges of a writer ascending and
 * adjacent (ra_log:handle_event/2 :849-896 ends at the highest index of the seq whose term matches, which
 * is what the ranges applied in ascending order leave), writers in the order given.  A writer takes at
 * most `max_per_row` (<= RA_LOCAL_CAP, minus what the caller reserves for other events of that row)
 * records of one step: the rest is reported through `resume` and goes into the next step.
 */
typedef struct ra_wal_writer {
    uint32_t row;                 /* the member (UId) the WAL wrote for                      */
    uint32_t n_ranges;
    uint64_t term;                /* #batch_writer.term                                      */
    const uint64_t* ranges;       /* n_ranges x {from, to}, ascending, non-overlapping       */
} ra_wal_writer;
typedef struct ra_wal_resume { uint32_t writer, range; } ra_wal_resume;   /* first range not emitted */
/* returns the number of events written to `out` (<= cap); *resume = {n_writers, 0} when the batch is done.
 * Start with *resume = {0, 0}; call again (next step) while resume->writer < n_writers. */
size_t ra_wal_batch_to_events(const ra_wal_writer* writers, size_t n_writers, uint32_t max_per_row,
                              ra_event* out, size_t cap, ra_wal_resume* resume);

/*
 * The same flood driven from the HOST through ra_engine_step (host buffers, H2D of the
 * step's events and D2H of its notes inside every step): what an Erlang batching process
 * in front of many ra_server_procs would do.  The host model (WAL completion, clients,
 * election timers) is the one ra_engine_flood runs on the device, so both paths leave
 * identical rows.  The engine must be route_on_device and freshly reset.
 */
typedef struct ra_hostsim ra_hostsim;
int  ra_hostsim_create(ra_engine* e, ra_hostsim** out);
/* the same over K engines holding disjoint sets of groups (partition p runs the model with seed + p): one
   host thread keeps all of them busy through ra_engine_submit_host / ra_engine_collect */
int  ra_hostsim_create_multi(ra_engine* const* engines, uint32_t n, ra_hostsim** out);
void ra_hostsim_destroy(ra_hostsim* s);
/* bootstrap != 0: first send election_timeout to slot 0 of every group (ra:trigger_election) */
int  ra_hostsim_run(ra_hostsim* s, uint32_t n_steps, uint32_t cmds_per_step,
                    uint32_t election_permille, uint64_t seed, int bootstrap);
/* bytes moved over PCIe by the last ra_hostsim_run and its wall time in seconds */
int  ra_hostsim_stats(ra_hostsim* s, uint64_t* h2d_bytes, uint64_t* d2h_bytes, double* seconds,
                      uint64_t* engine_calls);
/* where the wall time of the last run went: inside ra_engine_step vs in the host model */
int  ra_hostsim_breakdown(ra_hostsim* s, double* step_seconds, double* model_seconds);

/* pinned host memory for callers that want zero-copy staging of their batches */
void* ra_engine_alloc_host(size_t bytes);
void  ra_engine_free_host(void* p);

const char* ra_engine_strerror(int status);
const char* ra_engine_last_cuda_error(ra_engine* e);

#ifdef __cplusplus
}
#endif
#endif /* RA_ENGINE_H */
