/* TEST INFRASTRUCTURE: just enough of OTP's erl_nif.h (types and prototypes) to build
 * ra_b200/csrc/ra_engine_nif.c in an image without an Erlang toolchain.  tests/test_abi_exports.py::
 * test_nif_shim_compiles syntax-checks the shim against it; tests/nif_stub/erl_nif_stub.c implements the calls the shim
 * makes, and tests/test_nif_shim.py runs the shim through that implementation.  It is not the real header. */
#pragma once
#include <stddef.h>
#include <stdint.h>
typedef struct enif_environment_t ErlNifEnv;
typedef uintptr_t ERL_NIF_TERM;
typedef struct { size_t size; unsigned char* data; void* ref_bin; void* spare[2]; } ErlNifBinary;
typedef struct enif_resource_type_t ErlNifResourceType;
typedef void ErlNifResourceDtor(ErlNifEnv*, void*);
typedef enum { ERL_NIF_RT_CREATE = 1, ERL_NIF_RT_TAKEOVER = 2 } ErlNifResourceFlags;
typedef struct { const char* name; unsigned arity; ERL_NIF_TERM (*fptr)(ErlNifEnv*, int, const ERL_NIF_TERM[]); unsigned flags; } ErlNifFunc;
#define ERL_NIF_DIRTY_JOB_CPU_BOUND 1
ErlNifResourceType* enif_open_resource_type(ErlNifEnv*, const char*, const char*, ErlNifResourceDtor*, ErlNifResourceFlags, ErlNifResourceFlags*);
void* enif_alloc_resource(ErlNifResourceType*, size_t);
void enif_release_resource(void*);
ERL_NIF_TERM enif_make_resource(ErlNifEnv*, void*);
int enif_get_resource(ErlNifEnv*, ERL_NIF_TERM, ErlNifResourceType*, void**);
int enif_get_uint(ErlNifEnv*, ERL_NIF_TERM, unsigned*);
int enif_get_int(ErlNifEnv*, ERL_NIF_TERM, int*);
int enif_inspect_binary(ErlNifEnv*, ERL_NIF_TERM, ErlNifBinary*);
int enif_alloc_binary(size_t, ErlNifBinary*);
int enif_realloc_binary(ErlNifBinary*, size_t);
void enif_release_binary(ErlNifBinary*);
ERL_NIF_TERM enif_make_binary(ErlNifEnv*, ErlNifBinary*);
ERL_NIF_TERM enif_make_badarg(ErlNifEnv*);
ERL_NIF_TERM enif_make_atom(ErlNifEnv*, const char*);
ERL_NIF_TERM enif_make_int(ErlNifEnv*, int);
ERL_NIF_TERM enif_make_uint64(ErlNifEnv*, uint64_t);
ERL_NIF_TERM enif_make_tuple2(ErlNifEnv*, ERL_NIF_TERM, ERL_NIF_TERM);
ERL_NIF_TERM enif_make_new_map(ErlNifEnv*);
int enif_make_map_put(ErlNifEnv*, ERL_NIF_TERM, ERL_NIF_TERM, ERL_NIF_TERM, ERL_NIF_TERM*);
/* what the library hands the runtime: its module name, the NIF table and the load callback (as in OTP, nif_init) */
typedef struct {
    const char* name;
    int num_of_funcs;
    ErlNifFunc* funcs;
    int (*load)(ErlNifEnv*, void**, ERL_NIF_TERM);
} ErlNifEntry;
ErlNifEntry* nif_init(void);
#define ERL_NIF_INIT(MOD, FUNCS, LOAD, RELOAD, UPGRADE, UNLOAD) \
    ErlNifEntry* nif_init(void) \
    { static ErlNifEntry entry = { #MOD, (int)(sizeof(FUNCS) / sizeof(FUNCS[0])), FUNCS, LOAD }; return &entry; }
