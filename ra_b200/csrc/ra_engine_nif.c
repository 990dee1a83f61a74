/* ra_engine_nif.c -- dirty-NIF shim over include/ra_engine.h (see INTEGRATION.md).
 * The body is compiled only when the build defines RA_HAVE_ERL_NIF (with OTP's erl_nif.h).  Without an
 * OTP toolchain the test suite builds it against tests/nif_stub/ -- a header of the erl_nif API and a
 * working implementation of the calls made here -- and runs it against the oracle, on the host emulation
 * of the engine and on the engine itself (tests/test_nif_shim.py).
 * Records travel as binaries of the ABI structs (ra_event 64 B, ra_note 32 B, ra_row_state), which
 * the Erlang side builds / matches with bit syntax (INTEGRATION.md). */
#ifdef RA_HAVE_ERL_NIF
#include <erl_nif.h>
#include <string.h>
#include "../../include/ra_engine.h"

static ErlNifResourceType* ENG;

/* A submitted call whose buffers (a private copy of the events, the output binaries) must stay alive until it is
 * collected.  used = its submission number on this engine (0: free), rec = event record size, rc = a status collect
 * must return instead of collecting (its re-submission failed). */
typedef struct { ErlNifBinary ev, m, t; unsigned long used; size_t rec; int rc; } pend_t;

/* The engine resource: the engine and its calls in flight, two as in the engine.  Calls on one engine are serialised
 * by the caller (INTEGRATION.md, "Threading"), so nothing here needs a lock; calls on different engines share
 * nothing. */
typedef struct { ra_engine* e; pend_t pend[2]; unsigned long seq; } eng_t;

static pend_t* oldest_pend(eng_t* r)
{
    pend_t* p = NULL;
    for (int i = 0; i < 2; i++) if (r->pend[i].used && (!p || r->pend[i].used < p->used)) p = &r->pend[i];
    return p;
}

static void release_pend(pend_t* p)
{
    p->used = 0;
    enif_release_binary(&p->ev); enif_release_binary(&p->m); enif_release_binary(&p->t);
}

/* the last reference to the engine term is gone: wait for the calls still in flight, free their buffers, then the
 * engine */
static void eng_dtor(ErlNifEnv* env, void* obj)
{
    (void)env;
    eng_t* r = (eng_t*)obj;
    for (pend_t* p; (p = oldest_pend(r)) != NULL; ) {
        size_t nm, nn;
        if (!p->rc) (void)ra_engine_collect(r->e, &nm, &nn);
        release_pend(p);
    }
    ra_engine_destroy(r->e);
}

static int load(ErlNifEnv* env, void** priv, ERL_NIF_TERM info)
{
    (void)priv; (void)info;
    ENG = enif_open_resource_type(env, NULL, "ra_engine", eng_dtor, ERL_NIF_RT_CREATE, NULL);
    return ENG ? 0 : 1;
}

/* new(#{groups, members, device}) */
static ERL_NIF_TERM new_nif(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[])
{
    unsigned groups, members; int device;
    if (argc != 3 || !enif_get_uint(env, argv[0], &groups) || !enif_get_uint(env, argv[1], &members) ||
        !enif_get_int(env, argv[2], &device)) return enif_make_badarg(env);
    ra_engine_cfg cfg; memset(&cfg, 0, sizeof cfg);
    cfg.n_groups = groups; cfg.n_members = members; cfg.device = device;
    ra_engine* e = NULL;
    int rc = ra_engine_create(&cfg, &e);
    if (rc) return enif_make_tuple2(env, enif_make_atom(env, "error"), enif_make_int(env, rc));
    eng_t* r = (eng_t*)enif_alloc_resource(ENG, sizeof(eng_t));
    if (!r) { ra_engine_destroy(e); return enif_make_tuple2(env, enif_make_atom(env, "error"), enif_make_int(env, RA_E_NOMEM)); }
    memset(r, 0, sizeof *r);
    r->e = e;
    ERL_NIF_TERM t = enif_make_resource(env, r);
    enif_release_resource(r);
    return enif_make_tuple2(env, enif_make_atom(env, "ok"), t);
}

/* outputs of a finished call as {MsgsBin, NotesBin}.  n * CAP is only a first guess (rows without an event in
 * the batch emit too: deferred pipeline passes, mailbox records): when the engine answers RA_E_CAPACITY nothing
 * is lost -- the binaries are re-sized to what it reported and ra_engine_fetch_output takes the outputs. */
static ERL_NIF_TERM finish_outputs(ErlNifEnv* env, ra_engine* e, int rc, ErlNifBinary* m, ErlNifBinary* t,
                                   size_t nm, size_t nn)
{
    if (rc == RA_E_CAPACITY && (nm * sizeof(ra_event) > m->size || nn * sizeof(ra_note) > t->size)) {
        if (!enif_realloc_binary(m, (nm ? nm : 1) * sizeof(ra_event)) ||
            !enif_realloc_binary(t, (nn ? nn : 1) * sizeof(ra_note))) rc = RA_E_NOMEM;
        else rc = ra_engine_fetch_output(e, (ra_event*)m->data, m->size / sizeof(ra_event), &nm,
                                         (ra_note*)t->data, t->size / sizeof(ra_note), &nn);
    }
    if (rc) {
        enif_release_binary(m); enif_release_binary(t);
        return enif_make_tuple2(env, enif_make_atom(env, "error"), enif_make_int(env, rc));
    }
    enif_realloc_binary(m, nm * sizeof(ra_event));
    enif_realloc_binary(t, nn * sizeof(ra_note));
    return enif_make_tuple2(env, enif_make_binary(env, m), enif_make_binary(env, t));
}

/* step(Ref, EventsBin) / step_host(Ref, HostEventsBin) -> {MsgsBin, NotesBin} | {error, Code} */
static ERL_NIF_TERM step_any(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[], size_t rec)
{
    eng_t* r; ErlNifBinary ev;
    if (argc != 2 || !enif_get_resource(env, argv[0], ENG, (void**)&r) ||
        !enif_inspect_binary(env, argv[1], &ev) || ev.size % rec) return enif_make_badarg(env);
    size_t n = ev.size / rec, nm = 0, nn = 0;
    size_t mc = n * RA_MSG_CAP + 64, nc = n * RA_NOTE_CAP + 64;
    ErlNifBinary m, t;
    if (!enif_alloc_binary(mc * sizeof(ra_event), &m)) return enif_make_badarg(env);
    if (!enif_alloc_binary(nc * sizeof(ra_note), &t)) { enif_release_binary(&m); return enif_make_badarg(env); }
    int rc = rec == sizeof(ra_event)
        ? ra_engine_step(r->e, (const ra_event*)ev.data, n, (ra_event*)m.data, mc, &nm, (ra_note*)t.data, nc, &nn)
        : ra_engine_step_host(r->e, (const ra_host_event*)ev.data, n, (ra_event*)m.data, mc, &nm, (ra_note*)t.data, nc, &nn);
    return finish_outputs(env, r->e, rc, &m, &t, nm, nn);
}
static ERL_NIF_TERM step_nif(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[])
{ return step_any(env, argc, argv, sizeof(ra_event)); }
static ERL_NIF_TERM step_host_nif(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[])
{ return step_any(env, argc, argv, sizeof(ra_host_event)); }

static ERL_NIF_TERM status_term(ErlNifEnv* env, int rc)
{
    return rc ? enif_make_tuple2(env, enif_make_atom(env, "error"), enif_make_int(env, rc)) : enif_make_atom(env, "ok");
}

/* load_rows(Ref, RowsBin) -> ok | {error, Code}: RowsBin = << <<Row:sizeof(ra_row_state)/binary>> ... >> */
static ERL_NIF_TERM load_rows_nif(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[])
{
    eng_t* r; ErlNifBinary rows;
    if (argc != 2 || !enif_get_resource(env, argv[0], ENG, (void**)&r) ||
        !enif_inspect_binary(env, argv[1], &rows) || rows.size % sizeof(ra_row_state)) return enif_make_badarg(env);
    return status_term(env, ra_engine_load_rows(r->e, (const ra_row_state*)rows.data, rows.size / sizeof(ra_row_state)));
}

/* read_rows(Ref, RowIdsBin) -> RowsBin | {error, Code}: RowIdsBin = << <<Row:32/little>> ... >> */
static ERL_NIF_TERM read_rows_nif(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[])
{
    eng_t* r; ErlNifBinary ids, out;
    if (argc != 2 || !enif_get_resource(env, argv[0], ENG, (void**)&r) ||
        !enif_inspect_binary(env, argv[1], &ids) || ids.size % 4) return enif_make_badarg(env);
    const size_t n = ids.size / 4;
    if (!enif_alloc_binary(n * sizeof(ra_row_state), &out)) return enif_make_badarg(env);
    memset(out.data, 0, out.size);
    for (size_t i = 0; i < n; i++) memcpy(&((ra_row_state*)out.data)[i].row, ids.data + 4 * i, 4);
    int rc = ra_engine_read_rows(r->e, (ra_row_state*)out.data, n);
    if (rc) { enif_release_binary(&out); return status_term(env, rc); }
    return enif_make_binary(env, &out);
}

/* reset_empty(Ref) -> ok | {error, Code} */
static ERL_NIF_TERM reset_empty_nif(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[])
{
    eng_t* r;
    if (argc != 1 || !enif_get_resource(env, argv[0], ENG, (void**)&r)) return enif_make_badarg(env);
    return status_term(env, ra_engine_reset_empty(r->e));
}

/* counters(Ref) -> #{events => _, commits => _, ...} | {error, Code} */
static ERL_NIF_TERM counters_nif(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[])
{
    eng_t* r; ra_counters c;
    if (argc != 1 || !enif_get_resource(env, argv[0], ENG, (void**)&r)) return enif_make_badarg(env);
    int rc = ra_engine_counters(r->e, &c);
    if (rc) return status_term(env, rc);
    const char* names[] = {"events", "commits", "applied", "msgs_out", "msgs_dropped", "elections_won", "fatal_rows", "steps",
                           "aer_received_follower", "aer_received_follower_empty", "aer_replies_success",
                           "aer_replies_failed", "elections", "pre_vote_elections", "term_and_voted_for_updates"};
    const uint64_t vals[] = {c.events, c.commits, c.applied, c.msgs_out, c.msgs_dropped, c.elections_won, c.fatal_rows, c.steps,
                             c.aer_received_follower, c.aer_received_follower_empty, c.aer_replies_success,
                             c.aer_replies_failed, c.elections, c.pre_vote_elections, c.term_and_voted_for_updates};
    ERL_NIF_TERM map = enif_make_new_map(env);
    for (int i = 0; i < 15; i++)
        enif_make_map_put(env, map, enif_make_atom(env, names[i]), enif_make_uint64(env, vals[i]), &map);
    return map;
}

/* Split-phase calls.  The buffers of a submitted batch (a private copy of the events, the output binaries)
 * must stay alive until it is collected: they live in the engine resource (eng_t), two slots as in the engine.
 * submit(Ref, EventsBin) / submit_host(Ref, HostEventsBin) -> ok | {error, Code};
 * collect(Ref) -> {MsgsBin, NotesBin} | {error, Code}. */
static int submit_pend(ra_engine* e, pend_t* p)
{
    const size_t n = p->ev.size / p->rec, mc = p->m.size / sizeof(ra_event), nc = p->t.size / sizeof(ra_note);
    return p->rec == sizeof(ra_event)
        ? ra_engine_submit(e, (const ra_event*)p->ev.data, n, (ra_event*)p->m.data, mc, (ra_note*)p->t.data, nc)
        : ra_engine_submit_host(e, (const ra_host_event*)p->ev.data, n, (ra_event*)p->m.data, mc, (ra_note*)p->t.data, nc);
}

static ERL_NIF_TERM submit_any(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[], size_t rec)
{
    eng_t* r; ErlNifBinary ev;
    if (argc != 2 || !enif_get_resource(env, argv[0], ENG, (void**)&r) ||
        !enif_inspect_binary(env, argv[1], &ev) || ev.size % rec) return enif_make_badarg(env);
    pend_t* p = !r->pend[0].used ? &r->pend[0] : !r->pend[1].used ? &r->pend[1] : NULL;
    if (!p) return status_term(env, RA_E_BUSY);
    size_t n = ev.size / rec, mc = n * RA_MSG_CAP + 64, nc = n * RA_NOTE_CAP + 64;
    if (!enif_alloc_binary(ev.size ? ev.size : 1, &p->ev)) return status_term(env, RA_E_NOMEM);
    memcpy(p->ev.data, ev.data, ev.size);
    if (!enif_alloc_binary(mc * sizeof(ra_event), &p->m)) { enif_release_binary(&p->ev); return status_term(env, RA_E_NOMEM); }
    if (!enif_alloc_binary(nc * sizeof(ra_note), &p->t)) { enif_release_binary(&p->ev); enif_release_binary(&p->m); return status_term(env, RA_E_NOMEM); }
    p->rec = rec; p->rc = RA_OK;
    int rc = submit_pend(r->e, p);
    if (rc) { enif_release_binary(&p->ev); enif_release_binary(&p->m); enif_release_binary(&p->t); return status_term(env, rc); }
    p->used = ++r->seq;
    return status_term(env, RA_OK);
}
static ERL_NIF_TERM submit_nif(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[])
{ return submit_any(env, argc, argv, sizeof(ra_event)); }
static ERL_NIF_TERM submit_host_nif(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[])
{ return submit_any(env, argc, argv, sizeof(ra_host_event)); }

static ERL_NIF_TERM collect_nif(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[])
{
    eng_t* r;
    if (argc != 1 || !enif_get_resource(env, argv[0], ENG, (void**)&r)) return enif_make_badarg(env);
    pend_t* p = oldest_pend(r);                                  /* the oldest pending call of this engine */
    if (!p) return status_term(env, RA_E_INVAL);
    size_t nm = 0, nn = 0;
    int rc = p->rc ? p->rc : ra_engine_collect(r->e, &nm, &nn);
    p->used = 0;
    enif_release_binary(&p->ev);
    if (p->rc) { enif_release_binary(&p->m); enif_release_binary(&p->t); return status_term(env, rc); }
    /* outputs that did not fit: the call submitted behind this one was not evaluated (RA_E_PENDING).  Collect it,
     * fetch these outputs, then submit it again with its own buffers -- the caller's next collect returns it. */
    pend_t* q = rc == RA_E_CAPACITY ? oldest_pend(r) : NULL;
    int qrc = RA_OK;
    if (q) { size_t x, y; qrc = ra_engine_collect(r->e, &x, &y); }
    ERL_NIF_TERM out = finish_outputs(env, r->e, rc, &p->m, &p->t, nm, nn);
    if (q) q->rc = qrc == RA_E_PENDING ? submit_pend(r->e, q) : qrc;
    return out;
}

static ErlNifFunc funcs[] = {
    {"new", 3, new_nif, ERL_NIF_DIRTY_JOB_CPU_BOUND},
    {"load_rows", 2, load_rows_nif, ERL_NIF_DIRTY_JOB_CPU_BOUND},
    {"read_rows", 2, read_rows_nif, ERL_NIF_DIRTY_JOB_CPU_BOUND},
    {"reset_empty", 1, reset_empty_nif, ERL_NIF_DIRTY_JOB_CPU_BOUND},
    {"step", 2, step_nif, ERL_NIF_DIRTY_JOB_CPU_BOUND},
    {"step_host", 2, step_host_nif, ERL_NIF_DIRTY_JOB_CPU_BOUND},
    {"submit", 2, submit_nif, ERL_NIF_DIRTY_JOB_CPU_BOUND},
    {"submit_host", 2, submit_host_nif, ERL_NIF_DIRTY_JOB_CPU_BOUND},
    {"collect", 1, collect_nif, ERL_NIF_DIRTY_JOB_CPU_BOUND},
    {"counters", 1, counters_nif, ERL_NIF_DIRTY_JOB_CPU_BOUND},
};
ERL_NIF_INIT(ra_engine_nif, funcs, load, NULL, NULL, NULL)
#else
typedef int ra_engine_nif_not_built_without_erl_nif_h;
#endif
