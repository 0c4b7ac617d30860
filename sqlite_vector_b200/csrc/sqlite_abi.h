/*
 * sqlite_abi.h — the slice of SQLite's loadable-extension ABI that vector_ext.c uses.
 *
 * SQLite hands a loadable extension a table of function pointers (sqlite3_api_routines); its
 * layout is positional and append-only, so an extension only needs the POSITIONS of the entries it
 * calls.  tools/gen_sqlite_abi.py derives those positions from any SQLite sqlite3ext.h
 * (tests/test_sql_surface.py re-checks them against the amalgamation header when one is present).
 * The public structs below (sqlite3_module, sqlite3_index_info, sqlite3_vtab, sqlite3_vtab_cursor)
 * are the documented virtual-table interface: https://www.sqlite.org/vtab.html
 *
 * This replaces `#include "sqlite3ext.h"` + SQLITE_EXTENSION_INIT1/2 of the reference
 * (/root/reference/src/sqlite-vector.h:11-15, src/sqlite-vector.c:49-51, 2556-2558).
 */
#ifndef VSQ_SQLITE_ABI_H
#define VSQ_SQLITE_ABI_H

#include <stdarg.h>
#include <stdint.h>

typedef struct sqlite3 sqlite3;
typedef struct sqlite3_stmt sqlite3_stmt;
typedef struct sqlite3_value sqlite3_value;
typedef struct sqlite3_context sqlite3_context;
typedef long long sqlite3_int64;
typedef unsigned long long sqlite3_uint64;
typedef struct sqlite3_module sqlite3_module;
typedef struct sqlite3_vtab sqlite3_vtab;
typedef struct sqlite3_vtab_cursor sqlite3_vtab_cursor;
typedef struct sqlite3_index_info sqlite3_index_info;
typedef void (*sqlite3_destructor_type)(void *);

#define SQLITE_OK 0
#define SQLITE_ERROR 1
#define SQLITE_NOMEM 7
#define SQLITE_MISUSE 21
#define SQLITE_ROW 100
#define SQLITE_DONE 101
#define SQLITE_INTEGER 1
#define SQLITE_FLOAT 2
#define SQLITE_TEXT 3
#define SQLITE_BLOB 4
#define SQLITE_NULL 5
#define SQLITE_UTF8 1
#define SQLITE_STATIC ((sqlite3_destructor_type)0)
#define SQLITE_TRANSIENT ((sqlite3_destructor_type)-1)
#define SQLITE_INDEX_CONSTRAINT_EQ 2

struct sqlite3_vtab {
    const sqlite3_module *pModule;
    int nRef;
    char *zErrMsg;
};
struct sqlite3_vtab_cursor {
    sqlite3_vtab *pVtab;
};
struct sqlite3_index_info {
    int nConstraint;
    struct sqlite3_index_constraint {
        int iColumn;
        unsigned char op;
        unsigned char usable;
        int iTermOffset;
    } *aConstraint;
    int nOrderBy;
    struct sqlite3_index_orderby {
        int iColumn;
        unsigned char desc;
    } *aOrderBy;
    struct sqlite3_index_constraint_usage {
        int argvIndex;
        unsigned char omit;
    } *aConstraintUsage;
    int idxNum;
    char *idxStr;
    int needToFreeIdxStr;
    int orderByConsumed;
    double estimatedCost;
    sqlite3_int64 estimatedRows;
    int idxFlags;
    sqlite3_uint64 colUsed;
};
struct sqlite3_module {
    int iVersion;
    int (*xCreate)(sqlite3 *, void *, int, const char *const *, sqlite3_vtab **, char **);
    int (*xConnect)(sqlite3 *, void *, int, const char *const *, sqlite3_vtab **, char **);
    int (*xBestIndex)(sqlite3_vtab *, sqlite3_index_info *);
    int (*xDisconnect)(sqlite3_vtab *);
    int (*xDestroy)(sqlite3_vtab *);
    int (*xOpen)(sqlite3_vtab *, sqlite3_vtab_cursor **);
    int (*xClose)(sqlite3_vtab_cursor *);
    int (*xFilter)(sqlite3_vtab_cursor *, int, const char *, int, sqlite3_value **);
    int (*xNext)(sqlite3_vtab_cursor *);
    int (*xEof)(sqlite3_vtab_cursor *);
    int (*xColumn)(sqlite3_vtab_cursor *, sqlite3_context *, int);
    int (*xRowid)(sqlite3_vtab_cursor *, sqlite3_int64 *);
    int (*xUpdate)(sqlite3_vtab *, int, sqlite3_value **, sqlite3_int64 *);
    int (*xBegin)(sqlite3_vtab *);
    int (*xSync)(sqlite3_vtab *);
    int (*xCommit)(sqlite3_vtab *);
    int (*xRollback)(sqlite3_vtab *);
    int (*xFindFunction)(sqlite3_vtab *, int, const char *, void (**)(sqlite3_context *, int, sqlite3_value **), void **);
    int (*xRename)(sqlite3_vtab *, const char *);
    int (*xSavepoint)(sqlite3_vtab *, int);
    int (*xRelease)(sqlite3_vtab *, int);
    int (*xRollbackTo)(sqlite3_vtab *, int);
    int (*xShadowName)(const char *);
    int (*xIntegrity)(sqlite3_vtab *, const char *, const char *, int, char **);
};

/* positions inside sqlite3_api_routines (tools/gen_sqlite_abi.py) */
enum {
    VSQ_bind_blob = 2, VSQ_bind_double = 3, VSQ_bind_int = 4, VSQ_bind_int64 = 5, VSQ_bind_text = 10,
    VSQ_column_blob = 19, VSQ_column_bytes = 20, VSQ_column_double = 27, VSQ_column_int = 28, VSQ_column_int64 = 29,
    VSQ_column_text = 36, VSQ_column_type = 38, VSQ_create_function = 45, VSQ_create_module = 47, VSQ_declare_vtab = 50,
    VSQ_errmsg = 53, VSQ_exec = 55, VSQ_finalize = 57, VSQ_free = 58, VSQ_get_autocommit = 60, VSQ_malloc = 68, VSQ_mprintf = 69, VSQ_reset = 77,
    VSQ_result_blob = 78, VSQ_result_double = 79, VSQ_result_error = 80, VSQ_result_int = 82, VSQ_result_int64 = 83,
    VSQ_result_null = 84, VSQ_result_text = 85, VSQ_result_value = 89, VSQ_step = 94, VSQ_total_changes = 97,
    VSQ_user_data = 101, VSQ_value_blob = 102, VSQ_value_bytes = 103, VSQ_value_double = 105, VSQ_value_int = 106,
    VSQ_value_int64 = 107, VSQ_value_text = 109, VSQ_value_type = 113, VSQ_vmprintf = 114, VSQ_prepare_v2 = 116,
    VSQ_result_error_code = 146, VSQ_context_db_handle = 149, VSQ_create_function_v2 = 162, VSQ_malloc64 = 197,
    VSQ_API_SLOTS_USED = 198
};

typedef struct sqlite3_api_routines {
    void (*slot[VSQ_API_SLOTS_USED])(void);
} sqlite3_api_routines;

extern const sqlite3_api_routines *vsq_api;
#define VSQ_CALL(name, type) ((type)vsq_api->slot[VSQ_##name])

/* sqlite3_aggregate_context (vector_rowid_set) is the struct's first member; the slot table above is pinned by
 * tests/golden/sqlite3_api_slots.json, this one by tests/golden/sqlite3_api_slot_aggregate.json (tests/test_filtered_host.py),
 * both taken from the same sqlite3ext.h */
#define VSQ_SLOT_AGGREGATE_CONTEXT 0
#define sqlite3_aggregate_context ((void *(*)(sqlite3_context *, int))vsq_api->slot[VSQ_SLOT_AGGREGATE_CONTEXT])

#define sqlite3_bind_blob VSQ_CALL(bind_blob, int (*)(sqlite3_stmt *, int, const void *, int, sqlite3_destructor_type))
#define sqlite3_bind_double VSQ_CALL(bind_double, int (*)(sqlite3_stmt *, int, double))
#define sqlite3_bind_int VSQ_CALL(bind_int, int (*)(sqlite3_stmt *, int, int))
#define sqlite3_bind_int64 VSQ_CALL(bind_int64, int (*)(sqlite3_stmt *, int, sqlite3_int64))
#define sqlite3_bind_text VSQ_CALL(bind_text, int (*)(sqlite3_stmt *, int, const char *, int, sqlite3_destructor_type))
#define sqlite3_column_blob VSQ_CALL(column_blob, const void *(*)(sqlite3_stmt *, int))
#define sqlite3_column_bytes VSQ_CALL(column_bytes, int (*)(sqlite3_stmt *, int))
#define sqlite3_column_double VSQ_CALL(column_double, double (*)(sqlite3_stmt *, int))
#define sqlite3_column_int VSQ_CALL(column_int, int (*)(sqlite3_stmt *, int))
#define sqlite3_column_int64 VSQ_CALL(column_int64, sqlite3_int64 (*)(sqlite3_stmt *, int))
#define sqlite3_column_text VSQ_CALL(column_text, const unsigned char *(*)(sqlite3_stmt *, int))
#define sqlite3_column_type VSQ_CALL(column_type, int (*)(sqlite3_stmt *, int))
#define sqlite3_create_function                                                                                     \
    VSQ_CALL(create_function, int (*)(sqlite3 *, const char *, int, int, void *, void (*)(sqlite3_context *, int, sqlite3_value **), \
                                      void (*)(sqlite3_context *, int, sqlite3_value **), void (*)(sqlite3_context *)))
#define sqlite3_create_function_v2                                                                                  \
    VSQ_CALL(create_function_v2, int (*)(sqlite3 *, const char *, int, int, void *, void (*)(sqlite3_context *, int, sqlite3_value **), \
                                         void (*)(sqlite3_context *, int, sqlite3_value **), void (*)(sqlite3_context *), void (*)(void *)))
#define sqlite3_create_module VSQ_CALL(create_module, int (*)(sqlite3 *, const char *, const sqlite3_module *, void *))
#define sqlite3_declare_vtab VSQ_CALL(declare_vtab, int (*)(sqlite3 *, const char *))
#define sqlite3_errmsg VSQ_CALL(errmsg, const char *(*)(sqlite3 *))
#define sqlite3_exec VSQ_CALL(exec, int (*)(sqlite3 *, const char *, int (*)(void *, int, char **, char **), void *, char **))
#define sqlite3_finalize VSQ_CALL(finalize, int (*)(sqlite3_stmt *))
#define sqlite3_free VSQ_CALL(free, void (*)(void *))
#define sqlite3_get_autocommit VSQ_CALL(get_autocommit, int (*)(sqlite3 *))
#define sqlite3_malloc VSQ_CALL(malloc, void *(*)(int))
#define sqlite3_malloc64 VSQ_CALL(malloc64, void *(*)(sqlite3_uint64))
#define sqlite3_mprintf VSQ_CALL(mprintf, char *(*)(const char *, ...))
#define sqlite3_vmprintf VSQ_CALL(vmprintf, char *(*)(const char *, va_list))
#define sqlite3_prepare_v2 VSQ_CALL(prepare_v2, int (*)(sqlite3 *, const char *, int, sqlite3_stmt **, const char **))
#define sqlite3_reset VSQ_CALL(reset, int (*)(sqlite3_stmt *))
#define sqlite3_result_blob VSQ_CALL(result_blob, void (*)(sqlite3_context *, const void *, int, sqlite3_destructor_type))
#define sqlite3_result_double VSQ_CALL(result_double, void (*)(sqlite3_context *, double))
#define sqlite3_result_error VSQ_CALL(result_error, void (*)(sqlite3_context *, const char *, int))
#define sqlite3_result_error_code VSQ_CALL(result_error_code, void (*)(sqlite3_context *, int))
#define sqlite3_result_int VSQ_CALL(result_int, void (*)(sqlite3_context *, int))
#define sqlite3_result_int64 VSQ_CALL(result_int64, void (*)(sqlite3_context *, sqlite3_int64))
#define sqlite3_result_null VSQ_CALL(result_null, void (*)(sqlite3_context *))
#define sqlite3_result_text VSQ_CALL(result_text, void (*)(sqlite3_context *, const char *, int, sqlite3_destructor_type))
#define sqlite3_result_value VSQ_CALL(result_value, void (*)(sqlite3_context *, sqlite3_value *))
#define sqlite3_step VSQ_CALL(step, int (*)(sqlite3_stmt *))
#define sqlite3_total_changes VSQ_CALL(total_changes, int (*)(sqlite3 *))
#define sqlite3_user_data VSQ_CALL(user_data, void *(*)(sqlite3_context *))
#define sqlite3_value_blob VSQ_CALL(value_blob, const void *(*)(sqlite3_value *))
#define sqlite3_value_bytes VSQ_CALL(value_bytes, int (*)(sqlite3_value *))
#define sqlite3_value_double VSQ_CALL(value_double, double (*)(sqlite3_value *))
#define sqlite3_value_int VSQ_CALL(value_int, int (*)(sqlite3_value *))
#define sqlite3_value_int64 VSQ_CALL(value_int64, sqlite3_int64 (*)(sqlite3_value *))
#define sqlite3_value_text VSQ_CALL(value_text, const unsigned char *(*)(sqlite3_value *))
#define sqlite3_value_type VSQ_CALL(value_type, int (*)(sqlite3_value *))
#define sqlite3_context_db_handle VSQ_CALL(context_db_handle, sqlite3 *(*)(sqlite3_context *))

#endif /* VSQ_SQLITE_ABI_H */
