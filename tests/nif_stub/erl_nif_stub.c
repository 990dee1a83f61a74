/* TEST INFRASTRUCTURE: a working implementation of the erl_nif calls ra_b200/csrc/ra_engine_nif.c makes, so that the
 * dirty-NIF shim can be built and run without an Erlang runtime (tests/test_nif_shim.py drives it through ctypes, on the
 * host emulation of the engine and on the engine itself).  It models what the shim relies on:
 *
 *   terms      handles into a table of the env they were made in: integers, atoms (text kept per env), binaries,
 *              tuples, maps, resources and badarg;
 *   binaries   ERTS ownership: enif_alloc_binary gives the caller a binary, enif_make_binary hands it to the env and
 *              freeing the env frees it; a released binary is gone, and a reallocated one always moves, so that the
 *              old bytes are gone too.  Releasing a binary twice (or one the env owns) is counted, never done;
 *   resources  an atomic reference count: a resource term holds a reference while its env exists, a harness "keep"
 *              handle holds one until it is dropped, and the destructor runs when the last one goes, as the garbage
 *              collector would run it.
 *
 * Every count is atomic and every call is safe from several threads as long as each env is used by one thread at a
 * time (as an ErlNifEnv is).  The ra_stub_* functions at the end are the harness API for ctypes. */
#define _POSIX_C_SOURCE 200809L
#include <limits.h>
#include <pthread.h>
#include <stdalign.h>
#include <stdatomic.h>
#include <stdlib.h>
#include <string.h>
#include "erl_nif.h"

enum { K_NONE = 0, K_INT = 1, K_ATOM = 2, K_BIN = 3, K_TUPLE = 4, K_MAP = 5, K_RES = 6, K_BADARG = 7 };

static atomic_long live_bins, live_res, bad_releases, dtor_runs;

/* a binary's header: never freed (so that a second release can be recognised), its bytes are */
typedef struct { atomic_int live; unsigned char* data; size_t size; } bin_hdr;

struct enif_resource_type_t { ErlNifResourceDtor* dtor; };
typedef struct { ErlNifResourceType* type; atomic_long refs; alignas(max_align_t) unsigned char data[]; } res_hdr;
#define RES_OF(obj) ((res_hdr*)((unsigned char*)(obj) - offsetof(res_hdr, data)))

typedef struct {
    int kind;
    int is_unsigned;                 /* K_INT: the value is u (enif_make_uint64), else i */
    long long i;
    unsigned long long u;
    char* atom;
    bin_hdr* bin;
    ERL_NIF_TERM el[2];              /* K_TUPLE (arity 2) */
    size_t mn;                       /* K_MAP: mn pairs */
    ERL_NIF_TERM *mk, *mv;
    res_hdr* res;
} term;

struct enif_environment_t { term* t; size_t n, cap; };

static term* at(ErlNifEnv* env, ERL_NIF_TERM h) { return env && h >= 1 && h <= env->n ? &env->t[h - 1] : NULL; }

static ERL_NIF_TERM push(ErlNifEnv* env, term v)
{
    if (env->n == env->cap) {
        size_t cap = env->cap ? 2 * env->cap : 64;
        term* t = (term*)realloc(env->t, cap * sizeof(term));
        if (!t) abort();
        env->t = t; env->cap = cap;
    }
    env->t[env->n++] = v;
    return (ERL_NIF_TERM)env->n;
}

static ErlNifEnv* env_new(void) { return (ErlNifEnv*)calloc(1, sizeof(ErlNifEnv)); }

/* ---- binaries -------------------------------------------------------------------------------------------------- */
int enif_alloc_binary(size_t size, ErlNifBinary* bin)
{
    bin_hdr* h = (bin_hdr*)calloc(1, sizeof(bin_hdr));
    unsigned char* d = (unsigned char*)malloc(size ? size : 1);
    if (!h || !d) { free(h); free(d); return 0; }
    atomic_store(&h->live, 1);
    h->data = d; h->size = size;
    memset(bin, 0, sizeof *bin);
    bin->size = size; bin->data = d; bin->ref_bin = h;
    atomic_fetch_add(&live_bins, 1);
    return 1;
}

int enif_realloc_binary(ErlNifBinary* bin, size_t size)
{
    bin_hdr* h = (bin_hdr*)bin->ref_bin;
    if (!h || !atomic_load(&h->live)) { atomic_fetch_add(&bad_releases, 1); return 0; }
    unsigned char* d = (unsigned char*)malloc(size ? size : 1);
    if (!d) return 0;
    memcpy(d, h->data, size < h->size ? size : h->size);
    memset(h->data, 0xDB, h->size);                /* the old bytes are gone */
    free(h->data);
    h->data = d; h->size = size;
    bin->data = d; bin->size = size;
    return 1;
}

static void bin_release(bin_hdr* h)
{
    if (!h || atomic_exchange(&h->live, 0) != 1) { atomic_fetch_add(&bad_releases, 1); return; }
    memset(h->data, 0xDB, h->size);
    free(h->data);
    h->data = NULL;
    atomic_fetch_sub(&live_bins, 1);
}

void enif_release_binary(ErlNifBinary* bin) { bin_release((bin_hdr*)bin->ref_bin); }

ERL_NIF_TERM enif_make_binary(ErlNifEnv* env, ErlNifBinary* bin)
{
    term v; memset(&v, 0, sizeof v);
    v.kind = K_BIN; v.bin = (bin_hdr*)bin->ref_bin;
    if (!v.bin || !atomic_load(&v.bin->live)) atomic_fetch_add(&bad_releases, 1);
    return push(env, v);
}

int enif_inspect_binary(ErlNifEnv* env, ERL_NIF_TERM t, ErlNifBinary* bin)
{
    term* v = at(env, t);
    if (!v || v->kind != K_BIN) return 0;
    memset(bin, 0, sizeof *bin);
    bin->data = v->bin->data; bin->size = v->bin->size;    /* a view: ref_bin stays NULL, releasing it is a misuse */
    return 1;
}

/* ---- resources ------------------------------------------------------------------------------------------------- */
ErlNifResourceType* enif_open_resource_type(ErlNifEnv* env, const char* module, const char* name, ErlNifResourceDtor* dtor,
                                            ErlNifResourceFlags flags, ErlNifResourceFlags* tried)
{
    (void)env; (void)module; (void)name; (void)flags;
    if (tried) *tried = ERL_NIF_RT_CREATE;
    ErlNifResourceType* t = (ErlNifResourceType*)calloc(1, sizeof *t);
    if (t) t->dtor = dtor;
    return t;
}

void* enif_alloc_resource(ErlNifResourceType* type, size_t size)
{
    res_hdr* r = (res_hdr*)calloc(1, sizeof(res_hdr) + size);
    if (!r) return NULL;
    r->type = type;
    atomic_store(&r->refs, 1);
    atomic_fetch_add(&live_res, 1);
    return r->data;
}

static void env_free(ErlNifEnv* env);

void enif_release_resource(void* obj)
{
    res_hdr* r = RES_OF(obj);
    const long left = atomic_fetch_sub(&r->refs, 1) - 1;
    if (left < 0) { atomic_fetch_add(&bad_releases, 1); return; }
    if (left) return;
    if (r->type->dtor) {
        ErlNifEnv* env = env_new();
        r->type->dtor(env, obj);
        env_free(env);
    }
    atomic_fetch_add(&dtor_runs, 1);
    free(r);
    atomic_fetch_sub(&live_res, 1);
}

ERL_NIF_TERM enif_make_resource(ErlNifEnv* env, void* obj)
{
    term v; memset(&v, 0, sizeof v);
    v.kind = K_RES; v.res = RES_OF(obj);
    atomic_fetch_add(&v.res->refs, 1);
    return push(env, v);
}

int enif_get_resource(ErlNifEnv* env, ERL_NIF_TERM t, ErlNifResourceType* type, void** obj)
{
    term* v = at(env, t);
    if (!v || v->kind != K_RES || v->res->type != type) return 0;
    *obj = v->res->data;
    return 1;
}

/* ---- numbers, atoms, tuples, maps ------------------------------------------------------------------------------ */
static int get_ll(ErlNifEnv* env, ERL_NIF_TERM t, long long lo, unsigned long long hi, long long* out)
{
    term* v = at(env, t);
    if (!v || v->kind != K_INT) return 0;
    if (v->is_unsigned) { if (v->u > hi) return 0; *out = (long long)v->u; return 1; }
    if (v->i < lo || (v->i > 0 && (unsigned long long)v->i > hi)) return 0;
    *out = v->i;
    return 1;
}
int enif_get_uint(ErlNifEnv* env, ERL_NIF_TERM t, unsigned* out)
{ long long x; if (!get_ll(env, t, 0, UINT_MAX, &x)) return 0; *out = (unsigned)x; return 1; }
int enif_get_int(ErlNifEnv* env, ERL_NIF_TERM t, int* out)
{ long long x; if (!get_ll(env, t, INT_MIN, INT_MAX, &x)) return 0; *out = (int)x; return 1; }

ERL_NIF_TERM enif_make_int(ErlNifEnv* env, int i)
{ term v; memset(&v, 0, sizeof v); v.kind = K_INT; v.i = i; return push(env, v); }
ERL_NIF_TERM enif_make_uint64(ErlNifEnv* env, uint64_t u)
{ term v; memset(&v, 0, sizeof v); v.kind = K_INT; v.is_unsigned = 1; v.u = u; return push(env, v); }
ERL_NIF_TERM enif_make_badarg(ErlNifEnv* env)
{ term v; memset(&v, 0, sizeof v); v.kind = K_BADARG; return push(env, v); }

ERL_NIF_TERM enif_make_atom(ErlNifEnv* env, const char* name)
{
    term v; memset(&v, 0, sizeof v);
    v.kind = K_ATOM; v.atom = strdup(name);
    if (!v.atom) abort();
    return push(env, v);
}

ERL_NIF_TERM enif_make_tuple2(ErlNifEnv* env, ERL_NIF_TERM a, ERL_NIF_TERM b)
{ term v; memset(&v, 0, sizeof v); v.kind = K_TUPLE; v.el[0] = a; v.el[1] = b; return push(env, v); }

ERL_NIF_TERM enif_make_new_map(ErlNifEnv* env)
{ term v; memset(&v, 0, sizeof v); v.kind = K_MAP; return push(env, v); }

static int same_key(ErlNifEnv* env, ERL_NIF_TERM a, ERL_NIF_TERM b)
{
    term *x = at(env, a), *y = at(env, b);
    if (x->kind != y->kind) return 0;
    if (x->kind == K_ATOM) return strcmp(x->atom, y->atom) == 0;
    if (x->kind == K_INT) return x->is_unsigned == y->is_unsigned && x->i == y->i && x->u == y->u;
    return a == b;
}

int enif_make_map_put(ErlNifEnv* env, ERL_NIF_TERM map, ERL_NIF_TERM key, ERL_NIF_TERM value, ERL_NIF_TERM* out)
{
    term* m = at(env, map);
    if (!m || m->kind != K_MAP || !at(env, key) || !at(env, value)) return 0;
    term v; memset(&v, 0, sizeof v);
    v.kind = K_MAP;
    v.mk = (ERL_NIF_TERM*)malloc((m->mn + 1) * sizeof(ERL_NIF_TERM));
    v.mv = (ERL_NIF_TERM*)malloc((m->mn + 1) * sizeof(ERL_NIF_TERM));
    if (!v.mk || !v.mv) abort();
    int replaced = 0;
    for (size_t k = 0; k < m->mn; k++) {
        v.mk[k] = m->mk[k];
        v.mv[k] = m->mv[k];
        if (same_key(env, m->mk[k], key)) { v.mv[k] = value; replaced = 1; }
    }
    v.mn = m->mn;
    if (!replaced) { v.mk[v.mn] = key; v.mv[v.mn] = value; v.mn++; }
    *out = push(env, v);                 /* (m may have moved: push reallocates the table) */
    return 1;
}

/* ---- env ------------------------------------------------------------------------------------------------------- */
static void env_free(ErlNifEnv* env)
{
    if (!env) return;
    for (size_t k = 0; k < env->n; k++) {
        term* v = &env->t[k];
        if (v->kind == K_BIN && v->bin) bin_release(v->bin);
        else if (v->kind == K_ATOM) free(v->atom);
        else if (v->kind == K_MAP) { free(v->mk); free(v->mv); }
    }
    /* resources last: a destructor may release binaries of its own, never terms of this env */
    for (size_t k = 0; k < env->n; k++)
        if (env->t[k].kind == K_RES) enif_release_resource(env->t[k].res->data);
    free(env->t);
    free(env);
}

/* ---- harness API (ctypes) -------------------------------------------------------------------------------------- */
void* ra_stub_env_new(void) { return env_new(); }
void ra_stub_env_free(void* env) { env_free((ErlNifEnv*)env); }

ERL_NIF_TERM ra_stub_make_binary(void* env, const void* p, size_t n)
{
    ErlNifBinary b;
    if (!enif_alloc_binary(n, &b)) return 0;
    if (n) memcpy(b.data, p, n);
    return enif_make_binary((ErlNifEnv*)env, &b);
}
ERL_NIF_TERM ra_stub_make_int(void* env, long long i)
{ term v; memset(&v, 0, sizeof v); v.kind = K_INT; v.i = i; return push((ErlNifEnv*)env, v); }
ERL_NIF_TERM ra_stub_make_atom(void* env, const char* name) { return enif_make_atom((ErlNifEnv*)env, name); }
ERL_NIF_TERM ra_stub_make_resource(void* env, void* obj) { return enif_make_resource((ErlNifEnv*)env, obj); }

static pthread_once_t load_once = PTHREAD_ONCE_INIT;
static int load_rc = -1;
static void do_load(void)
{
    ErlNifEnv* env = env_new();
    void* priv = NULL;
    load_rc = nif_init()->load ? nif_init()->load(env, &priv, 0) : 0;
    env_free(env);
}
/* the runtime's load of the library: the shim's load callback, once */
int ra_stub_load(void) { pthread_once(&load_once, do_load); return load_rc; }

int ra_stub_nif_count(void) { return nif_init()->num_of_funcs; }
const char* ra_stub_nif_name(int k) { return nif_init()->funcs[k].name; }
unsigned ra_stub_nif_arity(int k) { return nif_init()->funcs[k].arity; }
unsigned ra_stub_nif_flags(int k) { return nif_init()->funcs[k].flags; }
const char* ra_stub_module(void) { return nif_init()->name; }

/* NAME/ARITY(argv) in env -> its result term, 0 when there is no such NIF */
ERL_NIF_TERM ra_stub_call(void* env, const char* name, unsigned arity, const ERL_NIF_TERM* argv)
{
    ra_stub_load();
    const ErlNifEntry* e = nif_init();
    for (int k = 0; k < e->num_of_funcs; k++)
        if (e->funcs[k].arity == arity && strcmp(e->funcs[k].name, name) == 0)
            return e->funcs[k].fptr((ErlNifEnv*)env, (int)arity, argv);
    return 0;
}

int ra_stub_kind(void* env, ERL_NIF_TERM t) { term* v = at((ErlNifEnv*)env, t); return v ? v->kind : K_NONE; }
int ra_stub_arity(void* env, ERL_NIF_TERM t) { term* v = at((ErlNifEnv*)env, t); return v && v->kind == K_TUPLE ? 2 : -1; }
ERL_NIF_TERM ra_stub_element(void* env, ERL_NIF_TERM t, int k)
{ term* v = at((ErlNifEnv*)env, t); return v && v->kind == K_TUPLE && k >= 0 && k < 2 ? v->el[k] : 0; }
/* the atom's text into buf (cap bytes, NUL-terminated) -> its length, -1 if t is no atom */
int ra_stub_atom_text(void* env, ERL_NIF_TERM t, char* buf, size_t cap)
{
    term* v = at((ErlNifEnv*)env, t);
    if (!v || v->kind != K_ATOM || !cap) return -1;
    strncpy(buf, v->atom, cap - 1);
    buf[cap - 1] = 0;
    return (int)strlen(v->atom);
}
/* -> 1: the value is *i, 2: the value is *u (enif_make_uint64), 0: no integer */
int ra_stub_integer(void* env, ERL_NIF_TERM t, long long* i, unsigned long long* u)
{
    term* v = at((ErlNifEnv*)env, t);
    if (!v || v->kind != K_INT) return 0;
    *i = v->i; *u = v->u;
    return v->is_unsigned ? 2 : 1;
}
int ra_stub_binary(void* env, ERL_NIF_TERM t, const unsigned char** data, size_t* size)
{
    term* v = at((ErlNifEnv*)env, t);
    if (!v || v->kind != K_BIN || !v->bin || !atomic_load(&v->bin->live)) return 0;
    *data = v->bin->data; *size = v->bin->size;
    return 1;
}
long long ra_stub_map_size(void* env, ERL_NIF_TERM t) { term* v = at((ErlNifEnv*)env, t); return v && v->kind == K_MAP ? (long long)v->mn : -1; }
ERL_NIF_TERM ra_stub_map_key(void* env, ERL_NIF_TERM t, size_t k)
{ term* v = at((ErlNifEnv*)env, t); return v && v->kind == K_MAP && k < v->mn ? v->mk[k] : 0; }
ERL_NIF_TERM ra_stub_map_value(void* env, ERL_NIF_TERM t, size_t k)
{ term* v = at((ErlNifEnv*)env, t); return v && v->kind == K_MAP && k < v->mn ? v->mv[k] : 0; }

/* a reference to the resource of term t that outlives t's env (a process holding the term), NULL if t is none */
void* ra_stub_keep(void* env, ERL_NIF_TERM t)
{
    term* v = at((ErlNifEnv*)env, t);
    if (!v || v->kind != K_RES) return NULL;
    atomic_fetch_add(&v->res->refs, 1);
    return v->res->data;
}
void ra_stub_drop(void* obj) { enif_release_resource(obj); }

long ra_stub_live_binaries(void) { return atomic_load(&live_bins); }
long ra_stub_live_resources(void) { return atomic_load(&live_res); }
long ra_stub_bad_releases(void) { return atomic_load(&bad_releases); }
long ra_stub_dtor_runs(void) { return atomic_load(&dtor_runs); }
