/*
 * vector_ext.c — SQLite loadable extension with sqlite-vector's SQL surface, scanning on the H100.
 *
 * Same entry point and SQL objects as the reference (src/sqlite-vector.c:2555-2638):
 *   scalar: vector_version, vector_backend, vector_init, vector_quantize (2|3 args), vector_quantize_memory,
 *           vector_quantize_preload, vector_quantize_cleanup, vector_as_{f32,f16,bf16,i8,u8} (1|2 args)
 *   table-valued: vector_full_scan, vector_quantize_scan (tbl, col, vector, k),
 *                 vector_full_scan_stream, vector_quantize_scan_stream (tbl, col, vector)
 * additions: vector_*_scan_batch (tbl, col, vectors, k); vector_*_scan_filtered (tbl, col, vector, k, rowids),
 *            vector_*_scan_batch_filtered (tbl, col, vectors, k, rowids) and the aggregate vector_rowid_set(x) that builds rowids;
 *            vector_*_scan_batch_sets (tbl, col, vectors, k, sets, query_sets) and the aggregate vector_rowid_sets(set, rowid);
 *            vector_*_scan_grouped (tbl, col, vector, k, groups, limit);
 *            vector_*_scan_range (tbl, col, vector, radius), vector_*_scan_range_filtered (tbl, col, vector, radius, rowids);
 *            vector_quantize_scan_rerank (tbl, col, vector, k, candidates), vector_quantize_scan_rerank_batch (tbl, col, vectors, k,
 *            candidates)
 * Column state, option parsing, JSON vectors, quantization build and the shadow-table chunk format are host
 * C and behave like the reference (citations at each function).  What differs is where a scan runs:
 *   vector_quantize_preload  -> chunks are staged through pinned memory into HBM (vsb_group_append_quant_chunk), row-sharded
 *                               over `gpus` GPUs (vector_init option gpus=N or env VSB_GPUS; default 1)
 *   vector_quantize_scan     -> vsb_group_scan_topk on the resident shards (replaces vQuantRun/vQuantRunMemory, :2121-2236)
 *   vector_full_scan         -> the raw column is staged to HBM on first use and re-staged when the
 *                               connection's change counters move (replaces vFullScanRun, :2071-2113)
 * There is no CPU scan: without a CUDA device the scan functions fail with the engine's error text.
 */
#define _GNU_SOURCE
#include <ctype.h>
#include <float.h>
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>

#include "sqlite_abi.h"
#include "vsb200.h"

const sqlite3_api_routines *vsq_api = 0;

#define VECTOR_EXT_VERSION "0.9.23-b200"
#define MAX_COLUMNS 128                        /* MAX_TABLES, src/sqlite-vector.c:72 */
#define DEFAULT_MAX_MEMORY (30 * 1024 * 1024)  /* src/sqlite-vector.c:71 */

/* the hidden columns every table-valued function starts with (src/sqlite-vector.c:98-103, :1830) */
enum { COL_TBL = 0, COL_VECTOR = 1, COL_K = 2, COL_MEMIDX = 3 };
#define N_MODULES 22                           /* rows of `modules`, the table-valued functions */

/* ------------------------------------------------------------------------------------------------ state */
/* the grouping of the most recent vector_*_scan_grouped statement on one staged column, with that statement's groups BLOB and its
 * dense key index -> user key mapping (DESIGN §3.15) */
typedef struct {
    vsb_grouping *gr;
    unsigned char *blob;
    sqlite3_int64 bytes;
    int64_t *keys;
} kept_grouping;

typedef struct {
    char *tbl, *col, *pk;          /* pk: "rowid" or the INTEGER PRIMARY KEY of a WITHOUT ROWID table */
    int vtype, dim, normalized, metric, qtype;
    int gpus;                      /* row shards (GPUs) the resident copies are spread over; option gpus=N / env VSB_GPUS, default 1 */
    uint64_t max_memory;
    float scale, offset;           /* quantization parameters (persisted in _sqliteai_vector) */
    vsb_group *qix;                /* resident quantized column: one shard per GPU (gpus = 1: a single shard) */
    int q_user_preloaded;          /* vector_quantize_preload was called (vs. staged lazily by a scan) */
    int q_tainted;                 /* lazily staged inside an open transaction: never reused (a ROLLBACK moves no counter) */
    sqlite3_int64 q_dataver;       /* PRAGMA data_version when the lazily staged copy was last verified */
    sqlite3_int64 q_fp[4];         /* shadow-table fingerprint at stage time: COUNT(*), SUM(counter), MIN(rowid1), MAX(rowid2) */
    vsb_group *fix;                /* resident raw column for vector_full_scan */
    sqlite3_int64 fix_dataver;
    int fix_changes;
    int fix_tainted;               /* staged inside an open transaction: never reused */
    kept_grouping q_kept, fix_kept; /* the grouped modules' kept grouping on qix / fix, freed before its column */
} vcolumn;

typedef struct module_def module_def;         /* one table-valued function: a row of `modules` */
typedef struct vcontext vcontext;
typedef struct {
    const module_def *def;
    vcontext *ctx;
} vmodule;                                     /* a module's pAux: its row and the connection's columns */
struct vcontext {
    vcolumn cols[MAX_COLUMNS];
    int ncols;
    vmodule mods[N_MODULES];
};

typedef struct {
    sqlite3_vtab base;
    sqlite3 *db;
    vcontext *ctx;
    const module_def *def;
} scan_vtab;

/* a result is ngroups groups of rows: group g has count[g] rows at ids / dist + g * stride and, for grouped scans, the key
 * key[g] of query query[g].  One group for the one-query modules, one per query for the many-query modules, one per returned key
 * (of every query) for grouped. */
typedef struct {
    sqlite3_vtab_cursor base;
    int64_t *ids;
    double *dist;
    float *fdist;                  /* a stream's distances, in place of dist: every row of the column is one result row */
    sqlite3_int64 *count, *key, *query;
    sqlite3_int64 ngroups, stride;
    sqlite3_int64 g, j;            /* the current row: row j of group g; a stream starts at j = -1, the reference's (0, 0.0) row */
    int max_index;                 /* carried from one xFilter to the next, as the reference's cursor does (:1808-1813) */
} scan_cursor;

/* ------------------------------------------------------------------------------------------------ helpers */
static int elem_size(int vtype) {
    switch (vtype) {
    case VSB_F32: return 4;
    case VSB_F16: case VSB_BF16: return 2;
    case VSB_U8: case VSB_I8: return 1;
    }
    return 0;
}
static const char *type_name(int vtype) { /* src/sqlite-vector.c:781-790 */
    switch (vtype) {
    case VSB_F32: return "FLOAT32";
    case VSB_F16: return "FLOAT16";
    case VSB_BF16: return "FLOATB16";
    case VSB_U8: return "UINT8";
    case VSB_I8: return "INT8";
    }
    return "N/A";
}
static int type_from_name(const char *s) { /* :772-779 */
    if (!strcasecmp(s, "FLOAT32")) return VSB_F32;
    if (!strcasecmp(s, "FLOAT16")) return VSB_F16;
    if (!strcasecmp(s, "FLOATB16")) return VSB_BF16;
    if (!strcasecmp(s, "UINT8")) return VSB_U8;
    if (!strcasecmp(s, "INT8")) return VSB_I8;
    return 0;
}
static int metric_from_name(const char *s) { /* :798-808 */
    if (!strcasecmp(s, "L2") || !strcasecmp(s, "EUCLIDEAN")) return VSB_L2;
    if (!strcasecmp(s, "SQUARED_L2")) return VSB_SQUARED_L2;
    if (!strcasecmp(s, "COSINE")) return VSB_COSINE;
    if (!strcasecmp(s, "DOT") || !strcasecmp(s, "INNER")) return VSB_DOT;
    if (!strcasecmp(s, "L1") || !strcasecmp(s, "MANHATTAN")) return VSB_L1;
    return 0;
}
static const char *sql_type_name(int t) { /* :241-249 */
    switch (t) {
    case SQLITE_TEXT: return "TEXT";
    case SQLITE_INTEGER: return "INTEGER";
    case SQLITE_FLOAT: return "REAL";
    case SQLITE_BLOB: return "BLOB";
    }
    return "N/A";
}

static float f32_of_bits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static uint32_t bits_of_f32(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static float bf16_to_f32(uint16_t h) { return f32_of_bits((uint32_t)h << 16); }
static uint16_t f32_to_bf16(float f) { /* RNE bit trick, src/distance-cpu.h:103-108 */
    uint32_t x = bits_of_f32(f);
    return (uint16_t)((x + 0x7FFFu + ((x >> 16) & 1u)) >> 16);
}
static float f16_to_f32(uint16_t h) { /* IEEE binary16 -> binary32, exact */
    uint32_t sign = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 0x1Fu, m = h & 0x3FFu;
    if (e == 0x1Fu) return f32_of_bits(sign | 0x7F800000u | (m << 13));
    if (e) return f32_of_bits(sign | ((e + 112u) << 23) | (m << 13));
    if (!m) return f32_of_bits(sign);
    int sh = 0;
    while (!(m & 0x400u)) { m <<= 1; ++sh; }
    return f32_of_bits(sign | ((uint32_t)(113 - sh) << 23) | ((m & 0x3FFu) << 13));
}
static uint16_t f32_to_f16(float f) { /* IEEE binary32 -> binary16, round to nearest even */
    uint32_t x = bits_of_f32(f), ax = x & 0x7FFFFFFFu;
    uint16_t sign = (uint16_t)((x >> 16) & 0x8000u);
    if (ax > 0x7F800000u) return (uint16_t)(sign | 0x7E00u);
    if (ax >= 0x47800000u) return (uint16_t)(sign | 0x7C00u);
    if (ax >= 0x38800000u) {
        uint32_t mant = ax & 0x7FFFFFu, h = (((ax >> 23) - 112u) << 10) | (mant >> 13), rem = mant & 0x1FFFu;
        if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) ++h;
        return (uint16_t)(sign | h);
    }
    if (ax < 0x33000000u) return sign;
    uint32_t mant = (ax & 0x7FFFFFu) | 0x800000u;
    int shift = 126 - (int)(ax >> 23);
    uint32_t h = mant >> shift, rem = mant & ((1u << shift) - 1u), half = 1u << (shift - 1);
    if (rem > half || (rem == half && (h & 1u))) ++h;
    return (uint16_t)(sign | h);
}

static char *dup_str(const char *s) {
    if (!s) return 0;
    size_t n = strlen(s) + 1;
    char *r = (char *)sqlite3_malloc((int)n);
    if (r) memcpy(r, s, n);
    return r;
}

static void fn_error(sqlite3_context *ctx, int rc, const char *fmt, ...) { /* context_result_error, :225-239 */
    char buf[4096];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    sqlite3_result_error(ctx, buf, -1);
    sqlite3_result_error_code(ctx, rc);
}
static int vtab_error(sqlite3_vtab *vt, const char *fmt, ...) { /* sqlite_vtab_set_error, :375-383 */
    va_list ap;
    va_start(ap, fmt);
    char *msg = sqlite3_vmprintf(fmt, ap);
    va_end(ap);
    if (vt->zErrMsg) sqlite3_free(vt->zErrMsg);
    vt->zErrMsg = msg;
    return SQLITE_ERROR;
}

static sqlite3_int64 query_int64(sqlite3 *db, const char *sql) { /* sqlite_read_int64, :385-397 */
    sqlite3_int64 v = 0;
    sqlite3_stmt *st = 0;
    if (sqlite3_prepare_v2(db, sql, -1, &st, 0) == SQLITE_OK && sqlite3_step(st) == SQLITE_ROW) v = sqlite3_column_int64(st, 0);
    sqlite3_finalize(st);
    return v;
}

static int check_args(sqlite3_context *ctx, const char *fname, int argc, sqlite3_value **argv, int want, const int *types) {
    /* sanity_check_args, :861-876 */
    if (argc != want) {
        fn_error(ctx, SQLITE_ERROR, "Function '%s' expects %d arguments, but %d were provided.", fname, want, argc);
        return 0;
    }
    for (int i = 0; i < argc; ++i) {
        int t = sqlite3_value_type(argv[i]);
        if (t != types[i]) {
            fn_error(ctx, SQLITE_ERROR, "Function '%s': argument %d must be of type %s (got %s).", fname, i + 1, sql_type_name(types[i]), sql_type_name(t));
            return 0;
        }
    }
    return 1;
}

/* ------------------------------------------------------------------------------------------------ catalog checks */
static int sys_exists(sqlite3 *db, const char *name, const char *type) { /* :191-215 */
    char *sql = sqlite3_mprintf("SELECT EXISTS (SELECT 1 FROM sqlite_master WHERE type='%q' AND name=? COLLATE NOCASE);", type);
    if (!sql) return 0;
    sqlite3_stmt *st = 0;
    int found = 0;
    if (sqlite3_prepare_v2(db, sql, -1, &st, 0) == SQLITE_OK) {
        sqlite3_bind_text(st, 1, name, -1, SQLITE_STATIC);
        if (sqlite3_step(st) == SQLITE_ROW) found = sqlite3_column_int(st, 0) != 0;
    }
    sqlite3_finalize(st);
    sqlite3_free(sql);
    return found;
}
static int column_exists(sqlite3 *db, const char *tbl, const char *col) { /* :270-285 */
    char *sql = sqlite3_mprintf("SELECT EXISTS(SELECT 1 FROM pragma_table_info('%q') WHERE name = ?1);", tbl);
    if (!sql) return 0;
    sqlite3_stmt *st = 0;
    int found = 0;
    if (sqlite3_prepare_v2(db, sql, -1, &st, 0) == SQLITE_OK) {
        sqlite3_bind_text(st, 1, col, -1, SQLITE_STATIC);
        if (sqlite3_step(st) == SQLITE_ROW) found = sqlite3_column_int(st, 0) != 0;
    }
    sqlite3_finalize(st);
    sqlite3_free(sql);
    return found;
}
static int column_is_blob(sqlite3 *db, const char *tbl, const char *col) { /* :287-305: no declared type counts as BLOB */
    char *sql = sqlite3_mprintf("SELECT type FROM pragma_table_info('%q') WHERE name=?", tbl);
    if (!sql) return 0;
    sqlite3_stmt *st = 0;
    int ok = 0;
    if (sqlite3_prepare_v2(db, sql, -1, &st, 0) == SQLITE_OK) {
        sqlite3_bind_text(st, 1, col, -1, SQLITE_STATIC);
        if (sqlite3_step(st) == SQLITE_ROW) {
            const char *t = (const char *)sqlite3_column_text(st, 0);
            ok = (t == 0) || strcasestr(t, "BLOB") != 0;
        }
    }
    sqlite3_finalize(st);
    sqlite3_free(sql);
    return ok;
}
static int table_without_rowid(sqlite3 *db, const char *tbl) { /* :307-323 */
    sqlite3_stmt *st = 0;
    int r = 0;
    if (sqlite3_prepare_v2(db, "SELECT sql FROM sqlite_master WHERE type='table' AND name=?", -1, &st, 0) == SQLITE_OK) {
        sqlite3_bind_text(st, 1, tbl, -1, SQLITE_STATIC);
        if (sqlite3_step(st) == SQLITE_ROW) {
            const char *s = (const char *)sqlite3_column_text(st, 0);
            r = s && strcasestr(s, "WITHOUT ROWID");
        }
    }
    sqlite3_finalize(st);
    return r;
}
static char *single_int_pk(sqlite3 *db, const char *tbl) { /* :325-348 */
    char *sql = sqlite3_mprintf("SELECT COUNT(*), type, name FROM pragma_table_info('%q') WHERE pk > 0;", tbl);
    if (!sql) return 0;
    sqlite3_stmt *st = 0;
    char *pk = 0;
    if (sqlite3_prepare_v2(db, sql, -1, &st, 0) == SQLITE_OK && sqlite3_step(st) == SQLITE_ROW && sqlite3_column_int(st, 0) == 1) {
        const char *decl = (const char *)sqlite3_column_text(st, 1);
        if (decl && strcasestr(decl, "INT")) pk = dup_str((const char *)sqlite3_column_text(st, 2));
    }
    sqlite3_finalize(st);
    sqlite3_free(sql);
    return pk;
}

/* ------------------------------------------------------------------------------------------------ options */
typedef struct {
    int vtype, dim, normalized, metric, qtype;
    int gpus;                      /* addition: 0 = not given */
    uint64_t max_memory;
} voptions;

static void options_default(voptions *o) { /* :1100-1106 */
    memset(o, 0, sizeof *o);
    o->vtype = VSB_F32;
    o->metric = VSB_L2;
    o->max_memory = DEFAULT_MAX_MEMORY;
    o->qtype = VSB_QUANT_AUTO;
}

static uint64_t parse_memory(const char *s) { /* human_to_number, :916-933 */
    char *end = 0;
    double d = strtod(s, &end);
    if (d == 0 || d == HUGE_VAL) return 0;
    while (*end && isspace((unsigned char)*end)) ++end;
    if (!strncasecmp(end, "KB", 2)) d *= 1024;
    else if (!strncasecmp(end, "MB", 2)) d *= 1024 * 1024;
    else if (!strncasecmp(end, "GB", 2)) d *= 1024.0 * 1024 * 1024;
    else if (*end) return 0;
    if (d < 0 || d > (double)INT64_MAX) return 0;
    return (uint64_t)d;
}

/* one key=value pair; keys match by case-insensitive PREFIX in this order, like :950-988 */
static int option_apply(sqlite3_context *ctx, voptions *o, const char *key, int klen, const char *val, int vlen) {
    if (klen == 0 || vlen == 0) return 0;
    char buf[256] = {0};
    memcpy(buf, val, (size_t)(vlen > 255 ? 255 : vlen));
    if (!strncasecmp(key, "type", (size_t)klen)) {
        int t = type_from_name(buf);
        if (!t) { fn_error(ctx, SQLITE_ERROR, "Invalid vector type: '%s' is not a recognized type.", buf); return 0; }
        o->vtype = t;
        return 1;
    }
    if (!strncasecmp(key, "dimension", (size_t)klen)) {
        int d = (int)strtol(buf, 0, 0);
        if (d <= 0) { fn_error(ctx, SQLITE_ERROR, "Invalid vector dimension: expected a positive integer, got '%s'.", buf); return 0; }
        o->dim = d;
        return 1;
    }
    if (!strncasecmp(key, "normalized", (size_t)klen)) { o->normalized = strtol(buf, 0, 0) != 0; return 1; }
    if (!strncasecmp(key, "max_memory", (size_t)klen)) { o->max_memory = (uint64_t)(int)parse_memory(buf); return 1; } /* int cast: :972 */
    if (!strncasecmp(key, "qtype", (size_t)klen)) {
        int q = !strcasecmp(buf, "UINT8") ? VSB_QUANT_U8 : (!strcasecmp(buf, "INT8") ? VSB_QUANT_S8 : -1);
        if (q < 0) { fn_error(ctx, SQLITE_ERROR, "Invalid quantization type: '%s' is not a recognized or supported quantization type.", buf); return 0; }
        o->qtype = q;
        return 1;
    }
    if (!strncasecmp(key, "distance", (size_t)klen)) {
        int m = metric_from_name(buf);
        if (!m) { fn_error(ctx, SQLITE_ERROR, "Invalid distance name: '%s' is not a recognized or supported distance.", buf); return 0; }
        o->metric = m;
        return 1;
    }
    if (!strncasecmp(key, "gpus", (size_t)klen)) {   /* addition (the reference ignores unknown keys, :990): row shards over N GPUs */
        int g = !strcasecmp(buf, "all") ? vsb_device_count() : (int)strtol(buf, 0, 0);
        if (g < 0) { fn_error(ctx, SQLITE_ERROR, "Invalid gpus value: expected a non-negative integer or 'all', got '%s'.", buf); return 0; }
        o->gpus = g;
        return 1;
    }
    return 1; /* unknown keys are ignored (:990) */
}

/* "k1=v1, k2=v2": malformed pairs are skipped (parse_keyvalue_string, :878-914) */
static int options_parse(sqlite3_context *ctx, const char *s, voptions *o) {
    if (!s) return 1;
    const char *p = s;
    while (*p) {
        while (*p && isspace((unsigned char)*p)) ++p;
        const char *k0 = p;
        while (*p && *p != '=' && *p != ',') ++p;
        int klen = (int)(p - k0);
        while (klen > 0 && isspace((unsigned char)k0[klen - 1])) --klen;
        if (*p != '=') {
            while (*p && *p != ',') ++p;
            if (*p == ',') ++p;
            continue;
        }
        ++p;
        while (*p && isspace((unsigned char)*p)) ++p;
        const char *v0 = p;
        while (*p && *p != ',') ++p;
        int vlen = (int)(p - v0);
        while (vlen > 0 && isspace((unsigned char)v0[vlen - 1])) --vlen;
        if (!option_apply(ctx, o, k0, klen, v0, vlen)) return 0;
        if (*p == ',') ++p;
    }
    return 1;
}

/* GPUs a column's resident copies are sharded over: option gpus=N, else env VSB_GPUS (N or "all"), else 1; never more than
 * the devices that are visible (the same SQL runs on a 1-GPU box) */
static int resolve_gpus(int opt) {
    int g = opt;
    if (g <= 0) {
        const char *e = getenv("VSB_GPUS");
        if (e && *e) g = !strcasecmp(e, "all") ? vsb_device_count() : atoi(e);
    }
    int have = vsb_device_count();
    const char *alias = getenv("VSB_GROUP_ALIAS");      /* tests: more shards than GPUs (see vsb_group_create) */
    if (g > have && !(alias && *alias && *alias != '0')) g = have;
    return g < 1 ? 1 : g;
}

/* ------------------------------------------------------------------------------------------------ context */
static vcolumn *ctx_find(vcontext *c, const char *tbl, const char *col) { /* vector_context_lookup, :1051-1061 */
    if (!tbl || !col) return 0;
    for (int i = 0; i < c->ncols; ++i) {
        vcolumn *v = &c->cols[i];
        if (v->tbl && v->col && !strcasecmp(v->tbl, tbl) && !strcasecmp(v->col, col)) return v;
    }
    return 0;
}
static void kept_free(kept_grouping *k) {
    vsb_grouping_free(k->gr);
    sqlite3_free(k->blob);
    sqlite3_free(k->keys);
    memset(k, 0, sizeof *k);
}
/* a staged column goes with the grouping kept on it */
static void drop_qix(vcolumn *v) {
    kept_free(&v->q_kept);
    vsb_group_free(v->qix);
    v->qix = 0;
}
static void drop_fix(vcolumn *v) {
    kept_free(&v->fix_kept);
    vsb_group_free(v->fix);
    v->fix = 0;
}
static void column_drop_device(vcolumn *v) {
    drop_qix(v);
    drop_fix(v);
    v->q_user_preloaded = 0;
}
static void ctx_free(void *p) { /* vector_context_free, :1038-1049 */
    vcontext *c = (vcontext *)p;
    if (!c) return;
    for (int i = 0; i < c->ncols; ++i) {
        column_drop_device(&c->cols[i]);
        sqlite3_free(c->cols[i].tbl);
        sqlite3_free(c->cols[i].col);
        sqlite3_free(c->cols[i].pk);
    }
    sqlite3_free(c);
}

/* reload qtype / qscale / qoffset persisted by a previous vector_quantize (sqlite_unserialize, :451-491) */
static void column_load_meta(sqlite3 *db, vcolumn *v) {
    sqlite3_stmt *st = 0;
    if (sqlite3_prepare_v2(db, "SELECT key, value FROM _sqliteai_vector WHERE tblname = ? AND colname = ?;", -1, &st, 0) != SQLITE_OK) {
        sqlite3_finalize(st);
        return;
    }
    sqlite3_bind_text(st, 1, v->tbl, -1, SQLITE_STATIC);
    sqlite3_bind_text(st, 2, v->col, -1, SQLITE_STATIC);
    while (sqlite3_step(st) == SQLITE_ROW) {
        const char *key = (const char *)sqlite3_column_text(st, 0);
        if (!key) continue;
        if (!strcmp(key, "qtype")) v->qtype = sqlite3_column_int(st, 1);
        else if (!strcmp(key, "qscale")) v->scale = (float)sqlite3_column_double(st, 1);
        else if (!strcmp(key, "qoffset")) v->offset = (float)sqlite3_column_double(st, 1);
    }
    sqlite3_finalize(st);
}
static int meta_store(sqlite3_context *ctx, const char *tbl, const char *col, const char *key, int is_int, sqlite3_int64 iv, double fv) {
    /* sqlite_serialize, :419-449 */
    sqlite3 *db = sqlite3_context_db_handle(ctx);
    sqlite3_stmt *st = 0;
    int rc = sqlite3_prepare_v2(db, "REPLACE INTO _sqliteai_vector (tblname, colname, key, value) VALUES (?, ?, ?, ?);", -1, &st, 0);
    if (rc == SQLITE_OK) {
        sqlite3_bind_text(st, 1, tbl, -1, SQLITE_STATIC);
        sqlite3_bind_text(st, 2, col, -1, SQLITE_STATIC);
        sqlite3_bind_text(st, 3, key, -1, SQLITE_STATIC);
        if (is_int) sqlite3_bind_int64(st, 4, iv);
        else sqlite3_bind_double(st, 4, fv);
        rc = sqlite3_step(st);
        if (rc == SQLITE_DONE) rc = SQLITE_OK;
    }
    if (rc != SQLITE_OK) sqlite3_result_error(ctx, sqlite3_errmsg(db), -1);
    sqlite3_finalize(st);
    return rc;
}

/* ------------------------------------------------------------------------------------------------ JSON vectors */
/* "[1, 2.5, ...]" -> blob of `vtype` elements (vector_from_json, :1528-1653).  Exactly one of ctx / vt is set. */
static void *json_to_blob(sqlite3_context *ctx, sqlite3_vtab *vt, int vtype, const char *json, int *out_size, int want_dim) {
#define JSON_FAIL(rc_, ...)                                     \
    do {                                                        \
        if (blob) sqlite3_free(blob);                           \
        if (vt) vtab_error(vt, __VA_ARGS__);                    \
        else if (ctx) fn_error(ctx, rc_, __VA_ARGS__);          \
        return 0;                                               \
    } while (0)
    char *blob = 0;
    while (*json && isspace((unsigned char)*json)) ++json;
    if (*json != '[') JSON_FAIL(SQLITE_ERROR, "Malformed JSON: expected '[' at the beginning of the array.");
    ++json;
    int commas = 0;
    for (const char *p = json; *p; ++p) commas += (*p == ',');
    const size_t es = (size_t)elem_size(vtype);
    const size_t alloc = (size_t)(commas + 1) * es;
    blob = (char *)sqlite3_malloc((int)alloc);
    if (!blob) JSON_FAIL(SQLITE_NOMEM, "Out of memory: unable to allocate %lld bytes for BLOB buffer.", (long long)alloc);
    int count = 0;
    const char *p = json;
    while (*p) {
        while (*p && isspace((unsigned char)*p)) ++p;
        if (*p == ']') break;
        char *end = 0;
        double v = strtod(p, &end);
        if (end == p) JSON_FAIL(SQLITE_ERROR, "Malformed JSON: expected a number at position %d (found '%c').", (int)(p - json) + 1, *p ? *p : '?');
        if (count >= (int)(alloc / es)) JSON_FAIL(SQLITE_ERROR, "Too many elements in JSON array.");
        switch (vtype) {
        case VSB_F32: ((float *)blob)[count++] = (float)v; break;
        case VSB_F16: ((uint16_t *)blob)[count++] = f32_to_f16((float)v); break;
        case VSB_BF16: ((uint16_t *)blob)[count++] = f32_to_bf16((float)v); break;
        case VSB_U8:
            if (v < 0 || v > 255) JSON_FAIL(SQLITE_ERROR, "Value out of range for uint8_t.");
            ((uint8_t *)blob)[count++] = (uint8_t)v;
            break;
        case VSB_I8:
            if (v < -128 || v > 127) JSON_FAIL(SQLITE_ERROR, "Value out of range for int8_t.");
            ((int8_t *)blob)[count++] = (int8_t)v;
            break;
        default: JSON_FAIL(SQLITE_ERROR, "Unsupported vector type.");
        }
        p = end;
        while (*p && isspace((unsigned char)*p)) ++p;
        if (*p == ',') {
            ++p;
            while (*p && isspace((unsigned char)*p)) ++p;
            if (*p == ']') break; /* trailing comma allowed */
        } else if (*p == ']') {
            break;
        } else {
            JSON_FAIL(SQLITE_ERROR, "Malformed JSON: unexpected character '%c' at position %d.", *p ? *p : '?', (int)(p - json) + 1);
        }
    }
    if (want_dim > 0 && want_dim != count) JSON_FAIL(SQLITE_ERROR, "Invalid JSON vector dimension: expected %d but found %d.", want_dim, count);
    if (out_size) *out_size = (int)((size_t)count * es);
    return blob;
#undef JSON_FAIL
}

/* vector_as_<type>(value [, dimension]) (vector_as_type, :1655-1699) */
static void as_type(sqlite3_context *ctx, int vtype, int argc, sqlite3_value **argv) {
    sqlite3_value *v = argv[0];
    int bytes = sqlite3_value_bytes(v), vt = sqlite3_value_type(v);
    int dim = (argc == 2) ? sqlite3_value_int(argv[1]) : 0;
    int es = elem_size(vtype);
    if (vt == SQLITE_BLOB) {
        if (bytes % es != 0) {
            fn_error(ctx, SQLITE_ERROR, "Invalid BLOB size for format '%s': size must be a multiple of %d bytes.", type_name(vtype), es);
            return;
        }
        if (dim > 0 && bytes != es * dim) {
            fn_error(ctx, SQLITE_ERROR, "Invalid BLOB size for format '%s': expected dimension should be %d (BLOB is %d bytes instead of %d).",
                     type_name(vtype), dim, bytes, es * dim);
            return;
        }
        sqlite3_result_value(ctx, v);
        return;
    }
    if (vt == SQLITE_TEXT) {
        const char *json = (const char *)sqlite3_value_text(v);
        if (!json) { fn_error(ctx, SQLITE_ERROR, "Invalid TEXT input."); return; }
        int size = 0;
        void *blob = json_to_blob(ctx, 0, vtype, json, &size, dim);
        if (blob) sqlite3_result_blob(ctx, blob, size, sqlite3_free);
        return;
    }
    fn_error(ctx, SQLITE_ERROR, "Unsupported input type: only BLOB and TEXT values are accepted (received %s).", sql_type_name(vt));
}
static void fn_as_f32(sqlite3_context *c, int n, sqlite3_value **a) { as_type(c, VSB_F32, n, a); }
static void fn_as_f16(sqlite3_context *c, int n, sqlite3_value **a) { as_type(c, VSB_F16, n, a); }
static void fn_as_bf16(sqlite3_context *c, int n, sqlite3_value **a) { as_type(c, VSB_BF16, n, a); }
static void fn_as_u8(sqlite3_context *c, int n, sqlite3_value **a) { as_type(c, VSB_U8, n, a); }
static void fn_as_i8(sqlite3_context *c, int n, sqlite3_value **a) { as_type(c, VSB_I8, n, a); }

/* ------------------------------------------------------------------------------------------------ quantizers */
static float elem_f32(int vtype, const void *v, int i) {
    switch (vtype) {
    case VSB_F32: return ((const float *)v)[i];
    case VSB_F16: return f16_to_f32(((const uint16_t *)v)[i]);
    case VSB_BF16: return bf16_to_f32(((const uint16_t *)v)[i]);
    case VSB_U8: return (float)((const uint8_t *)v)[i];
    case VSB_I8: return (float)((const int8_t *)v)[i];
    }
    return 0.0f;
}
/* q = round_half_away((v - offset) * scale), saturated.  f32 sources truncate an int cast and clamp
 * (src/sqlite-vector.c:517-548, 626-656); the other source types use the NaN/Inf-safe rounding of q_round_u8/s8 (:495-515). */
static void quantize_vec(int vtype, const void *v, uint8_t *q, float offset, float scale, int dim, int qtype) {
    for (int i = 0; i < dim; ++i) {
        float s = (elem_f32(vtype, v, i) - offset) * scale;
        float adj = 0.5f * (1.0f - 2.0f * (s < 0.0f));
        if (vtype == VSB_F32) {
            int r = (int)(s + adj);
            if (qtype == VSB_QUANT_U8) q[i] = (uint8_t)(r > 255 ? 255 : (r < 0 ? 0 : r));
            else ((int8_t *)q)[i] = (int8_t)(r > 127 ? 127 : (r < -128 ? -128 : r));
        } else if (qtype == VSB_QUANT_U8) {
            if (!isfinite(s)) q[i] = (s > 0.0f) ? 255u : 0u;
            else { float r = s + adj; q[i] = r >= 255.0f ? 255u : (r <= 0.0f ? 0u : (uint8_t)(int)r); }
        } else {
            if (!isfinite(s)) ((int8_t *)q)[i] = (s > 0.0f) ? 127 : (s < 0.0f ? -128 : 0);
            else { float r = s + adj; ((int8_t *)q)[i] = r >= 127.0f ? 127 : (r <= -128.0f ? -128 : (int8_t)(int)r); }
        }
    }
}

/* ------------------------------------------------------------------------------------------------ vector_init */
static void fn_version(sqlite3_context *ctx, int argc, sqlite3_value **argv) { (void)argc; (void)argv; sqlite3_result_text(ctx, VECTOR_EXT_VERSION, -1, SQLITE_STATIC); }
static void fn_backend(sqlite3_context *ctx, int argc, sqlite3_value **argv) { (void)argc; (void)argv; sqlite3_result_text(ctx, vsb_backend_name(), -1, SQLITE_TRANSIENT); }

static void fn_init(sqlite3_context *ctx, int argc, sqlite3_value **argv) { /* vector_init, :2491-2543 */
    static const int types[] = {SQLITE_TEXT, SQLITE_TEXT, SQLITE_TEXT};
    if (!check_args(ctx, "vector_init", argc, argv, 3, types)) return;
    const char *tbl = (const char *)sqlite3_value_text(argv[0]);
    const char *col = (const char *)sqlite3_value_text(argv[1]);
    const char *opts = (const char *)sqlite3_value_text(argv[2]);
    sqlite3 *db = sqlite3_context_db_handle(ctx);
    if (!sys_exists(db, tbl, "table")) { fn_error(ctx, SQLITE_ERROR, "Table '%s' does not exist.", tbl); return; }
    if (!column_exists(db, tbl, col)) { fn_error(ctx, SQLITE_ERROR, "Column '%s' does not exist in table '%s'.", col, tbl); return; }
    if (!column_is_blob(db, tbl, col)) { fn_error(ctx, SQLITE_ERROR, "Column '%s' in table '%s' must be of type BLOB.", col, tbl); return; }
    voptions o;
    options_default(&o);
    if (!options_parse(ctx, opts, &o)) return;
    if (o.vtype == 0) { fn_error(ctx, SQLITE_ERROR, "Vector type value is mandatory in vector_init"); return; }
    if (o.dim == 0) { fn_error(ctx, SQLITE_ERROR, "Vector dimension value is mandatory in vector_init"); return; }
    vcontext *vc = (vcontext *)sqlite3_user_data(ctx);
    vcolumn *v = ctx_find(vc, tbl, col);
    if (v) {
        if (o.dim != v->dim) { fn_error(ctx, SQLITE_ERROR, "Inconsistent vector dimension for '%s.%s': existing=%d, provided=%d.", tbl, col, v->dim, o.dim); return; }
        if (o.vtype != v->vtype) { fn_error(ctx, SQLITE_ERROR, "Inconsistent vector type for '%s.%s': existing=%s, provided=%s.", tbl, col, type_name(v->vtype), type_name(o.vtype)); return; }
        if (o.normalized != v->normalized) {
            fn_error(ctx, SQLITE_ERROR, "Inconsistent normalization flag for '%s.%s': existing=%s, provided=%s.", tbl, col, v->normalized ? "true" : "false", o.normalized ? "true" : "false");
            return;
        }
        if (o.gpus > 0 && o.gpus != v->gpus) { v->gpus = o.gpus; column_drop_device(v); }   /* re-sharded on the next preload / scan */
        return;
    }
    if (vc->ncols >= MAX_COLUMNS) { fn_error(ctx, SQLITE_ERROR, "Cannot add table: maximum number of allowed tables reached (%d).", MAX_COLUMNS); return; }
    char *t = dup_str(tbl), *c = dup_str(col);
    if (!t || !c) { sqlite3_free(t); sqlite3_free(c); fn_error(ctx, SQLITE_NOMEM, "Out of memory: unable to duplicate table or column name."); return; }
    int norowid = table_without_rowid(db, tbl);
    char *pk = norowid ? single_int_pk(db, tbl) : dup_str("rowid");
    if (!pk) {
        sqlite3_free(t); sqlite3_free(c);
        if (norowid) fn_error(ctx, SQLITE_ERROR, "WITHOUT ROWID table '%s' must have exactly one PRIMARY KEY column of type INTEGER.", tbl);
        else fn_error(ctx, SQLITE_NOMEM, "Out of memory: unable to duplicate rowid column name.");
        return;
    }
    v = &vc->cols[vc->ncols++];
    memset(v, 0, sizeof *v);
    v->tbl = t; v->col = c; v->pk = pk;
    v->vtype = o.vtype; v->dim = o.dim; v->normalized = o.normalized; v->metric = o.metric; v->qtype = o.qtype; v->max_memory = o.max_memory;
    v->gpus = o.gpus;
    column_load_meta(db, v);
}

/* ------------------------------------------------------------------------------------------------ quantize build */
static int flush_chunk(sqlite3 *db, const char *tbl, const char *col, uint32_t nrows, const uint8_t *data, size_t bytes, sqlite3_int64 lo, sqlite3_int64 hi) {
    /* one shadow-table row per chunk (vector_serialize_quantization, :1117-1145) */
    char *sql = sqlite3_mprintf("INSERT INTO vector0_%q_%q (rowid1, rowid2, counter, data) VALUES (?, ?, ?, ?);", tbl, col);
    if (!sql) return SQLITE_NOMEM;
    sqlite3_stmt *st = 0;
    int rc = sqlite3_prepare_v2(db, sql, -1, &st, 0);
    if (rc == SQLITE_OK) {
        sqlite3_bind_int64(st, 1, lo);
        sqlite3_bind_int64(st, 2, hi);
        sqlite3_bind_int(st, 3, (int)nrows);
        sqlite3_bind_blob(st, 4, data, (int)bytes, SQLITE_STATIC);
        rc = sqlite3_step(st);
        if (rc == SQLITE_DONE) rc = SQLITE_OK;
    }
    sqlite3_finalize(st);
    sqlite3_free(sql);
    return rc;
}

/* two passes over the column: global min/max, then [int64 LE rowid][dim x q8] rows packed into chunks of at most
 * max_memory bytes (vector_rebuild_quantization, :1147-1336) */
static int rebuild_quantization_host(sqlite3_context *ctx, vcolumn *v, int qtype, uint64_t max_memory, uint32_t *total) {
    sqlite3 *db = sqlite3_context_db_handle(ctx);
    const int dim = v->dim, vtype = v->vtype;
    const size_t qsize = 8 + (size_t)dim;
    *total = 0;
    if (max_memory == 0) {
        char *sql = sqlite3_mprintf("SELECT COUNT(*) FROM %q;", v->tbl);
        sqlite3_int64 count = sql ? query_int64(db, sql) : 0;
        sqlite3_free(sql);
        max_memory = (count == 0) ? DEFAULT_MAX_MEMORY : (uint64_t)count * qsize;
        if (count <= 0) {
            v->qtype = (qtype == VSB_QUANT_AUTO) ? VSB_QUANT_U8 : qtype;
            v->scale = 1.0f;
            v->offset = 0.0f;
            return SQLITE_OK;
        }
    }
    uint32_t max_vectors = (uint32_t)(max_memory / qsize);
    if (max_vectors == 0) max_vectors = 1;
    uint8_t *chunk = (uint8_t *)sqlite3_malloc64((sqlite3_uint64)max_vectors * qsize);
    if (!chunk) return SQLITE_NOMEM;
    char *sql = sqlite3_mprintf("SELECT %q, %q FROM %q ORDER BY %q;", v->pk, v->col, v->tbl, v->pk);
    sqlite3_stmt *st = 0;
    int rc = sql ? sqlite3_prepare_v2(db, sql, -1, &st, 0) : SQLITE_NOMEM;
    sqlite3_free(sql);
    if (rc != SQLITE_OK) goto done;

    float lo = FLT_MAX, hi = -FLT_MAX;
    int negative = 0;
    const size_t need = (size_t)dim * (size_t)elem_size(vtype);
    for (;;) {
        rc = sqlite3_step(st);
        if (rc == SQLITE_DONE) { rc = SQLITE_OK; break; }
        if (rc != SQLITE_ROW) goto done;
        if (sqlite3_column_type(st, 1) == SQLITE_NULL) continue;
        const void *blob = sqlite3_column_blob(st, 1);
        if (!blob) continue;
        if ((size_t)sqlite3_column_bytes(st, 1) < need) {
            fn_error(ctx, SQLITE_ERROR, "Invalid vector blob found at rowid %lld.", (long long)sqlite3_column_int64(st, 0));
            rc = SQLITE_ERROR;
            goto done;
        }
        for (int i = 0; i < dim; ++i) {
            float x = elem_f32(vtype, blob, i);
            if (x < lo) lo = x;
            if (x > hi) hi = x;
            if (x < 0.0) negative = 1;
        }
    }
    if (qtype == VSB_QUANT_AUTO) qtype = negative ? VSB_QUANT_S8 : VSB_QUANT_U8;      /* :1258-1261 */
    {
        float abs_max = fmaxf(fabsf(lo), fabsf(hi));
        v->scale = (qtype == VSB_QUANT_U8) ? (255.0f / (hi - lo)) : (127.0f / abs_max);  /* :1265-1268 */
        v->offset = (qtype == VSB_QUANT_U8) ? lo : 0.0f;
        v->qtype = qtype;
    }
    rc = sqlite3_reset(st);
    if (rc != SQLITE_OK) goto done;
    {
        uint32_t in_chunk = 0;
        sqlite3_int64 first_id = 0, last_id = 0;
        uint8_t *w = chunk;
        for (;;) {
            rc = sqlite3_step(st);
            if (rc == SQLITE_DONE) { rc = SQLITE_OK; break; }
            if (rc != SQLITE_ROW) goto done;
            if (sqlite3_column_type(st, 1) == SQLITE_NULL) continue;
            sqlite3_int64 id = sqlite3_column_int64(st, 0);
            const void *blob = sqlite3_column_blob(st, 1);
            if (!blob) continue;
            if (in_chunk == 0) first_id = id;
            for (int b = 0; b < 8; ++b) w[b] = (uint8_t)((uint64_t)id >> (8 * b));
            quantize_vec(vtype, blob, w + 8, v->offset, v->scale, dim, qtype);
            w += qsize;
            last_id = id;
            ++in_chunk;
            ++*total;
            if (in_chunk == max_vectors) {
                rc = flush_chunk(db, v->tbl, v->col, in_chunk, chunk, (size_t)(w - chunk), first_id, last_id);
                if (rc != SQLITE_OK) goto done;
                in_chunk = 0;
                w = chunk;
            }
        }
        if (in_chunk > 0) rc = flush_chunk(db, v->tbl, v->col, in_chunk, chunk, (size_t)(w - chunk), first_id, last_id);
    }
done:
    sqlite3_finalize(st);
    sqlite3_free(chunk);
    return rc;
}

/* what identifies the shadow table's current contents cheaply (vector_quantize rewrites every chunk) */
static void quant_fingerprint(sqlite3 *db, const vcolumn *v, sqlite3_int64 fp[4]) {
    fp[0] = fp[1] = fp[2] = fp[3] = -1;
    char *sql = sqlite3_mprintf("SELECT COUNT(*), SUM(counter), MIN(rowid1), MAX(rowid2) FROM vector0_%q_%q;", v->tbl, v->col);
    sqlite3_stmt *st = 0;
    if (sql && sqlite3_prepare_v2(db, sql, -1, &st, 0) == SQLITE_OK && sqlite3_step(st) == SQLITE_ROW)
        for (int i = 0; i < 4; ++i) fp[i] = sqlite3_column_int64(st, i);
    sqlite3_finalize(st);
    sqlite3_free(sql);
}

/* The same build with the two arithmetic loops on the GPU (vsb_quantizer_*): SQLite still steps through the rows and writes the
 * shadow table, the min / max reduction (:1224-1256) and the quantization into chunk bytes (:1281-1320) are kernels.  When the raw
 * column fits in HBM it is retained during pass 1 and the table is stepped ONCE (the reference steps it twice).  Output bytes,
 * chunk boundaries, rowid1 / rowid2 / counter columns and the stored scale / offset are identical (tests/golden/sql_surface.json). */
static int rebuild_quantization_gpu(sqlite3_context *ctx, vcolumn *v, int qtype, uint64_t max_memory, uint32_t *total) {
    sqlite3 *db = sqlite3_context_db_handle(ctx);
    const int dim = v->dim, vtype = v->vtype;
    const size_t qsize = 8 + (size_t)dim, need = (size_t)dim * (size_t)elem_size(vtype);
    *total = 0;
    char *sql = sqlite3_mprintf("SELECT COUNT(*) FROM %q;", v->tbl);
    sqlite3_int64 count = sql ? query_int64(db, sql) : 0;
    sqlite3_free(sql);
    if (max_memory == 0) {
        max_memory = (count == 0) ? DEFAULT_MAX_MEMORY : (uint64_t)count * qsize;
        if (count <= 0) {
            v->qtype = (qtype == VSB_QUANT_AUTO) ? VSB_QUANT_U8 : qtype;
            v->scale = 1.0f;
            v->offset = 0.0f;
            return SQLITE_OK;
        }
    }
    uint32_t max_vectors = (uint32_t)(max_memory / qsize);
    if (max_vectors == 0) max_vectors = 1;
    const int64_t block_rows = (int64_t)((4u << 20) / need) + 1;
    vsb_quantizer *qz = 0;
    uint8_t *block = 0, *chunk = 0;
    int64_t *ids = 0;
    size_t ids_cap = 0, nrows = 0;
    sqlite3_stmt *st = 0;
    int rc = SQLITE_OK;
    if (vsb_quantizer_create(&qz, 0, vtype, dim, count) != VSB_OK) { fn_error(ctx, SQLITE_ERROR, "vector_quantize: %s", vsb_last_error()); return SQLITE_ERROR; }
    block = (uint8_t *)malloc((size_t)block_rows * need);
    chunk = (uint8_t *)malloc((size_t)max_vectors * qsize);
    if (!block || !chunk) { rc = SQLITE_NOMEM; goto done; }
    sql = sqlite3_mprintf("SELECT %q, %q FROM %q ORDER BY %q;", v->pk, v->col, v->tbl, v->pk);
    rc = sql ? sqlite3_prepare_v2(db, sql, -1, &st, 0) : SQLITE_NOMEM;
    sqlite3_free(sql);
    if (rc != SQLITE_OK) goto done;
    {   /* pass 1: min / max on the GPU, rowids remembered on the host */
        int64_t nb = 0;
        for (;;) {
            rc = sqlite3_step(st);
            if (rc == SQLITE_DONE) { rc = SQLITE_OK; break; }
            if (rc != SQLITE_ROW) goto done;
            if (sqlite3_column_type(st, 1) == SQLITE_NULL) continue;
            const void *blob = sqlite3_column_blob(st, 1);
            if (!blob) continue;
            if ((size_t)sqlite3_column_bytes(st, 1) < need) {
                fn_error(ctx, SQLITE_ERROR, "Invalid vector blob found at rowid %lld.", (long long)sqlite3_column_int64(st, 0));
                rc = SQLITE_ERROR;
                goto done;
            }
            if (nrows == ids_cap) {
                size_t cap = ids_cap ? ids_cap * 2 : 65536;
                int64_t *p = (int64_t *)realloc(ids, cap * sizeof(int64_t));
                if (!p) { rc = SQLITE_NOMEM; goto done; }
                ids = p; ids_cap = cap;
            }
            ids[nrows++] = sqlite3_column_int64(st, 0);
            memcpy(block + (size_t)nb * need, blob, need);
            if (++nb == block_rows) {
                if (vsb_quantizer_minmax(qz, block, nb) != VSB_OK) { fn_error(ctx, SQLITE_ERROR, "vector_quantize: %s", vsb_last_error()); rc = SQLITE_ERROR; goto done; }
                nb = 0;
            }
        }
        if (nb > 0 && vsb_quantizer_minmax(qz, block, nb) != VSB_OK) { fn_error(ctx, SQLITE_ERROR, "vector_quantize: %s", vsb_last_error()); rc = SQLITE_ERROR; goto done; }
    }
    {
        float lo, hi;
        int negative = 0;
        if (vsb_quantizer_minmax_result(qz, &lo, &hi, &negative) != VSB_OK) { fn_error(ctx, SQLITE_ERROR, "vector_quantize: %s", vsb_last_error()); rc = SQLITE_ERROR; goto done; }
        if (qtype == VSB_QUANT_AUTO) qtype = negative ? VSB_QUANT_S8 : VSB_QUANT_U8;      /* :1258-1261 */
        float abs_max = fmaxf(fabsf(lo), fabsf(hi));
        v->scale = (qtype == VSB_QUANT_U8) ? (255.0f / (hi - lo)) : (127.0f / abs_max);  /* :1265-1268 */
        v->offset = (qtype == VSB_QUANT_U8) ? lo : 0.0f;
        v->qtype = qtype;
    }
    if (vsb_quantizer_retained_rows(qz) == (int64_t)nrows) {
        /* pass 2 from HBM: the raw column stayed on the device */
        for (size_t a = 0; a < nrows; a += max_vectors) {
            size_t m = nrows - a < max_vectors ? nrows - a : max_vectors;
            if (vsb_quantizer_encode(qz, 0, (int64_t)a, ids + a, (int64_t)m, v->offset, v->scale, qtype, chunk) != VSB_OK) {
                fn_error(ctx, SQLITE_ERROR, "vector_quantize: %s", vsb_last_error()); rc = SQLITE_ERROR; goto done;
            }
            rc = flush_chunk(db, v->tbl, v->col, (uint32_t)m, chunk, m * qsize, ids[a], ids[a + m - 1]);
            if (rc != SQLITE_OK) goto done;
            *total += (uint32_t)m;
        }
    } else {
        /* pass 2 streaming: step through the table again, one chunk of raw rows at a time */
        uint8_t *raw = (uint8_t *)malloc((size_t)max_vectors * need);
        if (!raw) { rc = SQLITE_NOMEM; goto done; }
        rc = sqlite3_reset(st);
        size_t a = 0, m = 0;
        while (rc == SQLITE_OK) {
            int s = sqlite3_step(st);
            if (s != SQLITE_ROW && s != SQLITE_DONE) { rc = s; break; }
            int have = 0;
            if (s == SQLITE_ROW) {
                if (sqlite3_column_type(st, 1) == SQLITE_NULL) continue;
                const void *blob = sqlite3_column_blob(st, 1);
                if (!blob) continue;
                memcpy(raw + m * need, blob, need);
                ++m;
                have = 1;
            }
            if (m == max_vectors || (s == SQLITE_DONE && m > 0)) {
                if (vsb_quantizer_encode(qz, raw, 0, ids + a, (int64_t)m, v->offset, v->scale, qtype, chunk) != VSB_OK) {
                    fn_error(ctx, SQLITE_ERROR, "vector_quantize: %s", vsb_last_error()); rc = SQLITE_ERROR; break;
                }
                rc = flush_chunk(db, v->tbl, v->col, (uint32_t)m, chunk, m * qsize, ids[a], ids[a + m - 1]);
                *total += (uint32_t)m;
                a += m;
                m = 0;
            }
            (void)have;
            if (s == SQLITE_DONE) break;
        }
        free(raw);
    }
done:
    sqlite3_finalize(st);
    vsb_quantizer_free(qz);
    free(block); free(chunk); free(ids);
    return rc;
}

/* GPU when a device is present (the product path; the -m gpu tests assert its kernels ran), else the host loops: the build is not
 * the scan hot path and a database must stay quantizable on a machine that only prepares it */
static int rebuild_quantization(sqlite3_context *ctx, vcolumn *v, int qtype, uint64_t max_memory, uint32_t *total) {
    const char *force = getenv("VSB_QUANTIZE_HOST");
    if (vsb_device_count() > 0 && !(force && *force == '1')) return rebuild_quantization_gpu(ctx, v, qtype, max_memory, total);
    return rebuild_quantization_host(ctx, v, qtype, max_memory, total);
}

/* stage every shadow-table chunk into HBM (the GPU counterpart of the loop at :1382-1394) */
static int stage_quantized(sqlite3 *db, vcolumn *v, char **errmsg) {
    drop_qix(v);
    v->q_tainted = !sqlite3_get_autocommit(db);
    v->q_dataver = query_int64(db, "PRAGMA data_version;");
    quant_fingerprint(db, v, v->q_fp);
    char *sql = sqlite3_mprintf("SELECT SUM(counter) FROM vector0_%q_%q;", v->tbl, v->col);
    sqlite3_int64 rows = sql ? query_int64(db, sql) : 0;
    sqlite3_free(sql);
    int rc = vsb_group_create(&v->qix, 0, resolve_gpus(v->gpus), v->qtype == VSB_QUANT_U8 ? VSB_U8 : VSB_I8, v->dim, rows);
    if (rc != VSB_OK) { *errmsg = sqlite3_mprintf("%s", vsb_last_error()); return SQLITE_ERROR; }
    sql = sqlite3_mprintf("SELECT counter, data FROM vector0_%q_%q;", v->tbl, v->col);
    sqlite3_stmt *st = 0;
    int src = sql ? sqlite3_prepare_v2(db, sql, -1, &st, 0) : SQLITE_NOMEM;
    sqlite3_free(sql);
    while (src == SQLITE_OK) {
        int s = sqlite3_step(st);
        if (s == SQLITE_DONE) break;
        if (s != SQLITE_ROW) { src = s; break; }
        sqlite3_int64 n = sqlite3_column_int64(st, 0);
        const void *data = sqlite3_column_blob(st, 1);
        if ((sqlite3_int64)sqlite3_column_bytes(st, 1) < n * (8 + (sqlite3_int64)v->dim)) { src = SQLITE_ERROR; *errmsg = sqlite3_mprintf("corrupt quantization chunk"); break; }
        rc = vsb_group_append_quant_chunk(v->qix, data, n);
        if (rc != VSB_OK) { src = SQLITE_ERROR; *errmsg = sqlite3_mprintf("%s", vsb_last_error()); break; }
    }
    sqlite3_finalize(st);
    if (src == SQLITE_OK && vsb_group_finalize(v->qix) != VSB_OK) { src = SQLITE_ERROR; *errmsg = sqlite3_mprintf("%s", vsb_last_error()); }
    if (src != SQLITE_OK) {
        if (!*errmsg) *errmsg = sqlite3_mprintf("%s", sqlite3_errmsg(db));
        drop_qix(v);
    }
    return src;
}

static void fn_quantize_preload(sqlite3_context *ctx, int argc, sqlite3_value **argv) { /* :1338-1404 */
    static const int types[] = {SQLITE_TEXT, SQLITE_TEXT};
    if (!check_args(ctx, "vector_quantize_preload", argc, argv, 2, types)) return;
    const char *tbl = (const char *)sqlite3_value_text(argv[0]);
    const char *col = (const char *)sqlite3_value_text(argv[1]);
    vcolumn *v = ctx_find((vcontext *)sqlite3_user_data(ctx), tbl, col);
    if (!v) {
        fn_error(ctx, SQLITE_ERROR, "Vector context not found for table '%s' and column '%s'. Ensure that vector_init() has been called before using vector_quantize_preload().", tbl, col);
        return;
    }
    sqlite3 *db = sqlite3_context_db_handle(ctx);
    char *sql = sqlite3_mprintf("SELECT SUM(LENGTH(data)) FROM vector0_%q_%q;", tbl, col);
    sqlite3_int64 required = sql ? query_int64(db, sql) : 0;
    sqlite3_free(sql);
    if (required == 0) {
        fn_error(ctx, SQLITE_ERROR, "Unable to read data from database. Ensure that vector_quantize() has been called before using vector_quantize_preload().");
        return;
    }
    char *err = 0;
    if (stage_quantized(db, v, &err) != SQLITE_OK) {
        fn_error(ctx, SQLITE_ERROR, "vector_quantize_preload: %s", err ? err : "device staging failed");
        sqlite3_free(err);
        return;
    }
    v->q_user_preloaded = 1;
}

static int do_quantize(sqlite3_context *ctx, const char *tbl, const char *col, const char *opts, int *was_preloaded) { /* :1406-1459 */
    vcolumn *v = ctx_find((vcontext *)sqlite3_user_data(ctx), tbl, col);
    if (!v) {
        fn_error(ctx, SQLITE_ERROR, "Vector context not found for table '%s' and column '%s'. Ensure that vector_init() has been called before using vector_quantize().", tbl, col);
        return SQLITE_ERROR;
    }
    sqlite3 *db = sqlite3_context_db_handle(ctx);
    uint32_t counter = 0;
    char *sql = 0;
    /* The reference brackets the rebuild with a bare BEGIN/COMMIT (:1418, :1446), which fails inside a caller's transaction
     * and then ROLLBACKs the caller's work.  A savepoint nests: deviation 9 in DESIGN.md. */
    int rc = sqlite3_exec(db, "SAVEPOINT vsb_quantize;", 0, 0, 0);
    if (rc != SQLITE_OK) { sqlite3_result_error_code(ctx, rc); return rc; }
    sql = sqlite3_mprintf("DROP TABLE IF EXISTS vector0_%q_%q;", tbl, col);
    rc = sql ? sqlite3_exec(db, sql, 0, 0, 0) : SQLITE_NOMEM;
    sqlite3_free(sql);
    if (rc != SQLITE_OK) goto fail;
    sql = sqlite3_mprintf("CREATE TABLE IF NOT EXISTS vector0_%q_%q (rowid1 INTEGER, rowid2 INTEGER, counter INTEGER, data BLOB);", tbl, col);
    rc = sql ? sqlite3_exec(db, sql, 0, 0, 0) : SQLITE_NOMEM;
    sqlite3_free(sql);
    if (rc != SQLITE_OK) goto fail;
    {
        voptions o;
        o.vtype = v->vtype; o.dim = v->dim; o.normalized = v->normalized; o.metric = v->metric; o.qtype = v->qtype; o.max_memory = v->max_memory;
        o.gpus = v->gpus;
        /* NOTE: like the reference (:1429), the options start from the column's CURRENT options, so a qtype chosen by an
         * earlier AUTO run sticks unless overridden */
        if (!options_parse(ctx, opts, &o)) {   /* the reference returns here with its transaction open (:1431); we undo the DROP */
            sqlite3_exec(db, "ROLLBACK TO vsb_quantize; RELEASE vsb_quantize;", 0, 0, 0);
            return SQLITE_ERROR;              /* options_parse has set the error message */
        }
        v->gpus = o.gpus;
        rc = rebuild_quantization(ctx, v, o.qtype, o.max_memory, &counter);
    }
    if (rc != SQLITE_OK) goto fail;
    rc = sqlite3_exec(db, "RELEASE vsb_quantize;", 0, 0, 0);
    if (rc != SQLITE_OK) goto fail;
    rc = meta_store(ctx, tbl, col, "qtype", 1, v->qtype, 0);
    if (rc == SQLITE_OK) rc = meta_store(ctx, tbl, col, "qscale", 0, 0, (double)v->scale);
    if (rc == SQLITE_OK) rc = meta_store(ctx, tbl, col, "qoffset", 0, 0, (double)v->offset);
    if (rc != SQLITE_OK) goto fail;
    *was_preloaded = v->q_user_preloaded;
    drop_qix(v);                                      /* the device copy is a cache of the shadow table */
    sqlite3_result_int64(ctx, (sqlite3_int64)counter);
    return SQLITE_OK;
fail:
    sqlite3_exec(db, "ROLLBACK TO vsb_quantize; RELEASE vsb_quantize;", 0, 0, 0);
    if (v->qix && !v->q_user_preloaded) drop_qix(v);
    sqlite3_result_error_code(ctx, rc);
    return rc;
}
static void fn_quantize3(sqlite3_context *ctx, int argc, sqlite3_value **argv) { /* :1461-1472 */
    static const int types[] = {SQLITE_TEXT, SQLITE_TEXT, SQLITE_TEXT};
    if (!check_args(ctx, "vector_quantize", argc, argv, 3, types)) return;
    int pre = 0;
    int rc = do_quantize(ctx, (const char *)sqlite3_value_text(argv[0]), (const char *)sqlite3_value_text(argv[1]), (const char *)sqlite3_value_text(argv[2]), &pre);
    if (rc == SQLITE_OK && pre) {
        /* the reference re-runs the preload, whose NULL result replaces the row count (:1471) */
        vcolumn *v = ctx_find((vcontext *)sqlite3_user_data(ctx), (const char *)sqlite3_value_text(argv[0]), (const char *)sqlite3_value_text(argv[1]));
        char *err = 0;
        if (v && stage_quantized(sqlite3_context_db_handle(ctx), v, &err) == SQLITE_OK) v->q_user_preloaded = 1;
        else { fn_error(ctx, SQLITE_ERROR, "vector_quantize_preload: %s", err ? err : "device staging failed"); }
        sqlite3_free(err);
    }
}
static void fn_quantize2(sqlite3_context *ctx, int argc, sqlite3_value **argv) { /* :1474-1484 */
    static const int types[] = {SQLITE_TEXT, SQLITE_TEXT};
    if (!check_args(ctx, "vector_quantize", argc, argv, 2, types)) return;
    int pre = 0;
    int rc = do_quantize(ctx, (const char *)sqlite3_value_text(argv[0]), (const char *)sqlite3_value_text(argv[1]), 0, &pre);
    if (rc == SQLITE_OK && pre) {
        vcolumn *v = ctx_find((vcontext *)sqlite3_user_data(ctx), (const char *)sqlite3_value_text(argv[0]), (const char *)sqlite3_value_text(argv[1]));
        char *err = 0;
        if (v && stage_quantized(sqlite3_context_db_handle(ctx), v, &err) == SQLITE_OK) v->q_user_preloaded = 1;
        else { fn_error(ctx, SQLITE_ERROR, "vector_quantize_preload: %s", err ? err : "device staging failed"); }
        sqlite3_free(err);
    }
}
static void fn_quantize_memory(sqlite3_context *ctx, int argc, sqlite3_value **argv) { /* :1486-1499 */
    static const int types[] = {SQLITE_TEXT, SQLITE_TEXT};
    if (!check_args(ctx, "vector_quantize_memory", argc, argv, 2, types)) return;
    char *sql = sqlite3_mprintf("SELECT SUM(LENGTH(data)) FROM vector0_%q_%q;", (const char *)sqlite3_value_text(argv[0]), (const char *)sqlite3_value_text(argv[1]));
    sqlite3_result_int64(ctx, sql ? query_int64(sqlite3_context_db_handle(ctx), sql) : 0);
    sqlite3_free(sql);
}
static void fn_quantize_cleanup(sqlite3_context *ctx, int argc, sqlite3_value **argv) { /* :1501-1524 */
    static const int types[] = {SQLITE_TEXT, SQLITE_TEXT};
    if (!check_args(ctx, "vector_quantize_cleanup", argc, argv, 2, types)) return;
    const char *tbl = (const char *)sqlite3_value_text(argv[0]);
    const char *col = (const char *)sqlite3_value_text(argv[1]);
    vcolumn *v = ctx_find((vcontext *)sqlite3_user_data(ctx), tbl, col);
    if (!v) return;
    drop_qix(v);
    v->q_user_preloaded = 0;
    char *sql = sqlite3_mprintf("DROP TABLE IF EXISTS vector0_%q_%q;", tbl, col);
    if (sql) sqlite3_exec(sqlite3_context_db_handle(ctx), sql, 0, 0, 0);
    sqlite3_free(sql);
}

/* ------------------------------------------------------------------------------------------------ raw column residency */
/* vector_full_scan reads the live table in the reference (SELECT pk, col FROM t; :2077).  Here the column is staged to
 * HBM and re-staged whenever this connection's change counter or the database's data_version moves. */
static int stage_full_column(scan_vtab *vt, vcolumn *v) {
    sqlite3 *db = vt->db;
    sqlite3_int64 dataver = query_int64(db, "PRAGMA data_version;");
    int changes = sqlite3_total_changes(db);
    /* Neither counter moves on ROLLBACK / ROLLBACK TO, so a copy staged while a transaction was open may hold rows that
     * were rolled back since: such a copy is used for the query that staged it and never again.  A copy staged in
     * autocommit mode holds committed rows only; it stays valid until a counter moves. */
    const int in_txn = !sqlite3_get_autocommit(db);
    if (v->fix && !v->fix_tainted && v->fix_dataver == dataver && v->fix_changes == changes) return SQLITE_OK;
    drop_fix(v);
    char *sql = sqlite3_mprintf("SELECT COUNT(*) FROM %q;", v->tbl);
    sqlite3_int64 total = sql ? query_int64(db, sql) : 0;
    sqlite3_free(sql);
    if (vsb_group_create(&v->fix, 0, resolve_gpus(v->gpus), v->vtype, v->dim, total) != VSB_OK) return vtab_error(&vt->base, "vector_full_scan: %s", vsb_last_error());
    sql = sqlite3_mprintf("SELECT %q, %q FROM %q;", v->pk, v->col, v->tbl);
    sqlite3_stmt *st = 0;
    int rc = sql ? sqlite3_prepare_v2(db, sql, -1, &st, 0) : SQLITE_NOMEM;
    sqlite3_free(sql);
    const size_t need = (size_t)v->dim * (size_t)elem_size(v->vtype);
    const int batch_rows = (int)((4u << 20) / need) + 1;
    uint8_t *rows = (uint8_t *)sqlite3_malloc64((sqlite3_uint64)batch_rows * need);
    sqlite3_int64 *ids = (sqlite3_int64 *)sqlite3_malloc64((sqlite3_uint64)batch_rows * sizeof(sqlite3_int64));
    if (!rows || !ids) rc = SQLITE_NOMEM;
    int nb = 0;
    while (rc == SQLITE_OK) {
        int s = sqlite3_step(st);
        if (s != SQLITE_ROW) { if (s != SQLITE_DONE) rc = s; break; }
        if (sqlite3_column_type(st, 1) == SQLITE_NULL) continue;           /* NULL rows are skipped (:2093) */
        const void *blob = sqlite3_column_blob(st, 1);
        if (!blob) continue;                                                 /* (:2096) */
        if ((size_t)sqlite3_column_bytes(st, 1) < need) {
            /* the reference reads past a short blob (SURVEY appendix B.7); we refuse instead */
            rc = vtab_error(&vt->base, "Invalid vector blob found at rowid %lld.", (long long)sqlite3_column_int64(st, 0));
            break;
        }
        memcpy(rows + (size_t)nb * need, blob, need);
        ids[nb++] = sqlite3_column_int64(st, 0);
        if (nb == batch_rows) {
            if (vsb_group_append_dense(v->fix, rows, (const int64_t *)ids, nb) != VSB_OK) { rc = vtab_error(&vt->base, "vector_full_scan: %s", vsb_last_error()); break; }
            nb = 0;
        }
    }
    if (rc == SQLITE_OK && nb > 0 && vsb_group_append_dense(v->fix, rows, (const int64_t *)ids, nb) != VSB_OK) rc = vtab_error(&vt->base, "vector_full_scan: %s", vsb_last_error());
    if (rc == SQLITE_OK && vsb_group_finalize(v->fix) != VSB_OK) rc = vtab_error(&vt->base, "vector_full_scan: %s", vsb_last_error());
    sqlite3_finalize(st);
    sqlite3_free(rows);
    sqlite3_free(ids);
    if (rc != SQLITE_OK) {
        drop_fix(v);
        if (!vt->base.zErrMsg) vtab_error(&vt->base, "vector_full_scan: %s", sqlite3_errmsg(db));
        return SQLITE_ERROR;
    }
    v->fix_dataver = dataver;
    v->fix_changes = changes;
    v->fix_tainted = in_txn;
    return SQLITE_OK;
}

/* ------------------------------------------------------------------------------------------------ virtual tables
 * Every table-valued function is one row of `modules`: the column it scans, one query or many, its hidden arguments after
 * memidx and its operation.  One xConnect, xFilter and cursor serve them all (vCursorFilterCommon, :1723-1826).  The reference
 * has vector_full_scan / vector_quantize_scan (tbl, col, vector, k) and their *_stream twins (tbl, col, vector); the rest are
 * additions without a counterpart there:
 *
 * vector_*_scan_batch(tbl, col, vectors, k): B queries in one call.  `vectors` is a BLOB of B x dimension elements of the column's
 *   type back to back, or a flat JSON array of B x dimension numbers.  Rows are (query, id, distance) with query = 0 .. B-1, each
 *   query's rows exactly those of the single-query function in the same order.  B >= 16 on F16/BF16/INT8/UINT8 data is scored on
 *   the tensor cores, except L1, which is batched on the CUDA cores for every column type (FLOAT32 too).
 * vector_*_scan_filtered(tbl, col, vector, k, rowids) / vector_*_scan_batch_filtered(tbl, col, vectors, k, rowids): the k nearest
 *   among the rows whose rowid is in `rowids`, a BLOB of little-endian int64 (vector_rowid_set builds it): the results of the
 *   unfiltered function over a table holding only those rows (vsb_group_scan_topk_filtered).
 * vector_*_scan_batch_sets(tbl, col, vectors, k, sets, query_sets): query b's k nearest among the rows of its own set.  `sets` is a
 *   BLOB of little-endian (int64 set, int64 rowid) pairs (vector_rowid_sets builds it); `query_sets` a BLOB of nq int64 set indexes
 *   (vector_rowid_set builds it), or NULL: query b uses set b.  Set indexes may be sparse; one that no pair names is an empty set.
 *   Each query's rows equal vector_*_scan_batch_filtered with that query's set (vsb_group_scan_topk_sets, DESIGN §3.14).
 * vector_*_scan_grouped(tbl, col, vector, k, groups, limit): each key's k nearest rows for the `limit` best keys (NULL or 0: every
 *   key with a row), keys ranked by their first row's distance, then its scan position, then the key.  `groups` is a BLOB of
 *   little-endian (int64 key, int64 rowid) pairs (vector_rowid_sets builds it); keys may be sparse.  Rows are (key, id, distance),
 *   keys in rank order and each key's rows exactly those of vector_*_scan_filtered with that key's rowids
 *   (vsb_group_scan_topk_grouped, DESIGN §3.15).  The reference answers it with row_number() OVER (PARTITION BY key ORDER BY
 *   distance) over vector_*_scan_stream.  Each of the two modules keeps the grouping (vsb_grouping_create) of its most recent
 *   statement beside the staged column it scanned, with a copy of that statement's groups BLOB and its key mapping: a statement
 *   whose groups BLOB is byte for byte the kept one, on the same staged column, skips the decoding of the BLOB and the layout.
 *   Anything else lays the keys out anew and replaces the kept grouping; re-staging the column (a changed table, data_version,
 *   or a copy staged inside a transaction) and closing the connection free it.  The rows returned are the same either way.
 * vector_*_scan_grouped_batch(tbl, col, vectors, k, groups, limit): B queries of vector_*_scan_grouped in one call, `vectors` as
 *   for vector_*_scan_batch.  Rows are (query, key, id, distance): query b's rows are exactly those vector_*_scan_grouped returns
 *   for vector b, queries in order.  The queries share each pass of the column (DESIGN §3.15); k = 0 returns no rows.  The two
 *   batch modules share the kept grouping of the column with the single ones: a repeated groups BLOB skips the layout whichever
 *   of them ran last.  Arguments are checked as for every module (test_sql_modules_host.py): the count, each argument in
 *   position order (k >= 0, the groups BLOB a whole number of pairs, limit >= 0), the context, the vectors, the quantization
 *   table and staging.
 * vector_*_scan_range(tbl, col, vector, radius) and the *_range_filtered twins (+ rowids): every row with distance < radius,
 *   ordered by distance, equal distances in scan order (vsb_group_scan_range).  The reference answers this only as
 *   SELECT id, distance FROM vector_*_scan_stream(...) WHERE distance < radius ORDER BY distance: the same rows, here without a
 *   pass of every row through the VM.  For vector_quantize_scan_range the radius is in the units vector_quantize_scan reports.
 *   The radius takes the hidden column `k`.
 * vector_quantize_scan_rerank(tbl, col, vector, k, candidates) / vector_quantize_scan_rerank_batch(tbl, col, vectors, k,
 *   candidates): the top `candidates` rows of the quantized column, reranked by their raw-column distance.  The single function
 *   returns row for row what
 *     SELECT id, distance FROM vector_full_scan_filtered(tbl, col, vector, k,
 *         (SELECT vector_rowid_set(id) FROM vector_quantize_scan(tbl, col, vector, candidates)))
 *   returns, but the rerank reads only the candidate rows of the raw column (vsb_group_scan_topk_rows) instead of all of it.  The
 *   batch function returns (query, id, distance), each query's rows those of the single function.  Distances are raw-column
 *   distances.  candidates may be smaller than k (fewer rows come back) or 0 (no rows). */
enum { OP_TOPK, OP_STREAM, OP_RANGE, OP_SETS, OP_GROUPED, OP_RERANK };
enum { ARG_NONE, ARG_TEXT, ARG_VECTOR, ARG_K, ARG_RADIUS, ARG_ROWIDS, ARG_SETS, ARG_QUERY_SETS, ARG_GROUPS, ARG_LIMIT, ARG_CANDIDATES };

struct module_def {
    const char *name, *schema;
    int quantized;                 /* scans the quantized column (rerank: for its candidates, then the raw column) */
    int many;                      /* `vector` holds B x dimension queries: one group of result rows per query */
    int hidden[2];                 /* the arguments after memidx (ARG_NONE: none) */
    int op;                        /* top-k (filtered: with rowids, batch: many), stream, range, sets, grouped or rerank */
};

#define SCHEMA(cols) "CREATE TABLE x(tbl hidden, vector hidden, k hidden, memidx hidden, " cols ");"
static const module_def modules[] = {
    {"vector_full_scan", SCHEMA("id, distance"), 0, 0, {ARG_NONE}, OP_TOPK},
    {"vector_quantize_scan", SCHEMA("id, distance"), 1, 0, {ARG_NONE}, OP_TOPK},
    {"vector_full_scan_stream", SCHEMA("id, distance"), 0, 0, {ARG_NONE}, OP_STREAM},
    {"vector_quantize_scan_stream", SCHEMA("id, distance"), 1, 0, {ARG_NONE}, OP_STREAM},
    {"vector_full_scan_batch", SCHEMA("query, id, distance"), 0, 1, {ARG_NONE}, OP_TOPK},
    {"vector_quantize_scan_batch", SCHEMA("query, id, distance"), 1, 1, {ARG_NONE}, OP_TOPK},
    {"vector_full_scan_filtered", SCHEMA("rowids hidden, id, distance"), 0, 0, {ARG_ROWIDS}, OP_TOPK},
    {"vector_quantize_scan_filtered", SCHEMA("rowids hidden, id, distance"), 1, 0, {ARG_ROWIDS}, OP_TOPK},
    {"vector_full_scan_batch_filtered", SCHEMA("rowids hidden, query, id, distance"), 0, 1, {ARG_ROWIDS}, OP_TOPK},
    {"vector_quantize_scan_batch_filtered", SCHEMA("rowids hidden, query, id, distance"), 1, 1, {ARG_ROWIDS}, OP_TOPK},
    {"vector_full_scan_batch_sets", SCHEMA("sets hidden, query_sets hidden, query, id, distance"), 0, 1, {ARG_SETS, ARG_QUERY_SETS}, OP_SETS},
    {"vector_quantize_scan_batch_sets", SCHEMA("sets hidden, query_sets hidden, query, id, distance"), 1, 1, {ARG_SETS, ARG_QUERY_SETS}, OP_SETS},
    {"vector_full_scan_grouped", SCHEMA("groups hidden, \"limit\" hidden, key, id, distance"), 0, 0, {ARG_GROUPS, ARG_LIMIT}, OP_GROUPED},
    {"vector_quantize_scan_grouped", SCHEMA("groups hidden, \"limit\" hidden, key, id, distance"), 1, 0, {ARG_GROUPS, ARG_LIMIT}, OP_GROUPED},
    {"vector_full_scan_grouped_batch", SCHEMA("groups hidden, \"limit\" hidden, query, key, id, distance"), 0, 1, {ARG_GROUPS, ARG_LIMIT}, OP_GROUPED},
    {"vector_quantize_scan_grouped_batch", SCHEMA("groups hidden, \"limit\" hidden, query, key, id, distance"), 1, 1, {ARG_GROUPS, ARG_LIMIT}, OP_GROUPED},
    {"vector_full_scan_range", SCHEMA("id, distance"), 0, 0, {ARG_NONE}, OP_RANGE},
    {"vector_quantize_scan_range", SCHEMA("id, distance"), 1, 0, {ARG_NONE}, OP_RANGE},
    {"vector_full_scan_range_filtered", SCHEMA("rowids hidden, id, distance"), 0, 0, {ARG_ROWIDS}, OP_RANGE},
    {"vector_quantize_scan_range_filtered", SCHEMA("rowids hidden, id, distance"), 1, 0, {ARG_ROWIDS}, OP_RANGE},
    {"vector_quantize_scan_rerank", SCHEMA("candidates hidden, id, distance"), 1, 0, {ARG_CANDIDATES}, OP_RERANK},
    {"vector_quantize_scan_rerank_batch", SCHEMA("candidates hidden, query, id, distance"), 1, 1, {ARG_CANDIDATES}, OP_RERANK},
};
#undef SCHEMA
_Static_assert(sizeof modules / sizeof modules[0] == N_MODULES, "N_MODULES counts the rows of modules");

static int nhidden(const module_def *m) { return (m->hidden[0] != ARG_NONE) + (m->hidden[1] != ARG_NONE); }
/* many-query and grouped results lead each row with its query or key, and number the rows by their position in the result */
static int leads_group(const module_def *m) { return m->many || m->op == OP_GROUPED; }
/* the columns before id: query and / or key (the batch grouped modules lead with both) */
static int lead_columns(const module_def *m) { return leads_group(m) + (m->many && m->op == OP_GROUPED); }

static int vt_connect(sqlite3 *db, void *aux, int argc, const char *const *argv, sqlite3_vtab **out, char **err) { /* :1828-1842 */
    (void)argc; (void)argv; (void)err;
    const vmodule *mod = (const vmodule *)aux;
    int rc = sqlite3_declare_vtab(db, mod->def->schema);
    if (rc != SQLITE_OK) return rc;
    scan_vtab *vt = (scan_vtab *)sqlite3_malloc((int)sizeof *vt);
    if (!vt) return SQLITE_NOMEM;
    memset(vt, 0, sizeof *vt);
    vt->db = db;
    vt->ctx = mod->ctx;
    vt->def = mod->def;
    *out = &vt->base;
    return SQLITE_OK;
}
static int vt_disconnect(sqlite3_vtab *p) { sqlite3_free(p); return SQLITE_OK; }

static void map_constraints(sqlite3_vtab *t, sqlite3_index_info *ii) { /* hidden column N -> argv[N] (:1856-1878) */
    const int last_hidden = COL_MEMIDX + nhidden(((scan_vtab *)t)->def);
    for (int i = 0; i < ii->nConstraint; ++i) {
        const struct sqlite3_index_constraint *c = &ii->aConstraint[i];
        if (!c->usable || c->op != SQLITE_INDEX_CONSTRAINT_EQ) continue;
        if (c->iColumn >= COL_TBL && c->iColumn <= last_hidden) {
            ii->aConstraintUsage[i].argvIndex = c->iColumn + 1;
            ii->aConstraintUsage[i].omit = 1;
        }
    }
}
static int vt_best_index_stream(sqlite3_vtab *t, sqlite3_index_info *ii) { /* :2245-2275 */
    ii->estimatedCost = 1e8;
    ii->estimatedRows = 100000;
    map_constraints(t, ii);
    return SQLITE_OK;
}
static int vt_best_index(sqlite3_vtab *t, sqlite3_index_info *ii) { /* :1850-1880 */
    if (((scan_vtab *)t)->def->op == OP_STREAM) return vt_best_index_stream(t, ii);
    ii->estimatedCost = 1.0;
    ii->estimatedRows = 100;
    ii->orderByConsumed = 1;
    ii->idxNum = 1;
    map_constraints(t, ii);
    return SQLITE_OK;
}

static int vt_open(sqlite3_vtab *t, sqlite3_vtab_cursor **out) {
    (void)t;
    scan_cursor *c = (scan_cursor *)sqlite3_malloc((int)sizeof *c);
    if (!c) return SQLITE_NOMEM;
    memset(c, 0, sizeof *c);
    *out = &c->base;
    return SQLITE_OK;
}
static void cursor_free_result(scan_cursor *c) {
    sqlite3_free(c->ids); sqlite3_free(c->dist); sqlite3_free(c->fdist); sqlite3_free(c->count); sqlite3_free(c->key);
    sqlite3_free(c->query);
    c->ids = 0; c->dist = 0; c->fdist = 0; c->count = 0; c->key = 0; c->query = 0;
}
static int vt_close(sqlite3_vtab_cursor *cur) {
    cursor_free_result((scan_cursor *)cur);
    sqlite3_free(cur);
    return SQLITE_OK;
}
/* the cursor's result arrays for `groups` groups of up to `stride` rows: float distances for a stream, a key and a query per group
 * for grouped */
static int cursor_alloc(scan_cursor *c, sqlite3_int64 groups, sqlite3_int64 stride, int op) {
    const sqlite3_uint64 ng = (sqlite3_uint64)(groups > 0 ? groups : 1), nr = ng * (sqlite3_uint64)(stride > 0 ? stride : 1);
    cursor_free_result(c);
    c->ids = (int64_t *)sqlite3_malloc64(nr * sizeof(int64_t));
    if (op == OP_STREAM) c->fdist = (float *)sqlite3_malloc64(nr * sizeof(float));
    else c->dist = (double *)sqlite3_malloc64(nr * sizeof(double));
    c->count = (sqlite3_int64 *)sqlite3_malloc64(ng * sizeof(sqlite3_int64));
    if (op == OP_GROUPED) {
        c->key = (sqlite3_int64 *)sqlite3_malloc64(ng * sizeof(sqlite3_int64));
        c->query = (sqlite3_int64 *)sqlite3_malloc64(ng * sizeof(sqlite3_int64));
    }
    c->stride = stride;
    return c->ids && (c->dist || c->fdist) && c->count && ((c->key && c->query) || op != OP_GROUPED) ? SQLITE_OK : SQLITE_NOMEM;
}
static void skip_empty(scan_cursor *c) {
    while (c->g < c->ngroups && c->j >= c->count[c->g]) { ++c->g; c->j = 0; }
}
static int vt_next(sqlite3_vtab_cursor *cur) {
    scan_cursor *c = (scan_cursor *)cur;
    ++c->j;
    skip_empty(c);
    return SQLITE_OK;
}
static int vt_eof(sqlite3_vtab_cursor *cur) {
    const scan_cursor *c = (const scan_cursor *)cur;
    return c->g >= c->ngroups;
}
static sqlite3_int64 cur_id(const scan_cursor *c) { return c->j < 0 ? 0 : c->ids[c->g * c->stride + c->j]; }
static int vt_column(sqlite3_vtab_cursor *cur, sqlite3_context *ctx, int col) { /* :2006-2014 */
    const scan_cursor *c = (const scan_cursor *)cur;
    const module_def *m = ((scan_vtab *)cur->pVtab)->def;
    const sqlite3_int64 at = c->g * c->stride + c->j;
    const int first = COL_MEMIDX + 1 + nhidden(m), lead = lead_columns(m);   /* the visible columns: [query,] [key,] id, distance */
    if (lead == 2 && col == first) sqlite3_result_int64(ctx, c->query[c->g]);
    else if (lead && col == first + lead - 1) sqlite3_result_int64(ctx, c->key ? c->key[c->g] : c->g);
    else if (col == first + lead) sqlite3_result_int64(ctx, cur_id(c));
    else if (col == first + lead + 1) sqlite3_result_double(ctx, c->j < 0 ? 0.0 : c->fdist ? (double)c->fdist[at] : c->dist[at]);
    return SQLITE_OK;
}
static int vt_rowid(sqlite3_vtab_cursor *cur, sqlite3_int64 *out) {
    const scan_cursor *c = (const scan_cursor *)cur;
    *out = leads_group(((scan_vtab *)cur->pVtab)->def) ? c->g * c->stride + c->j : cur_id(c);
    return SQLITE_OK;
}

/* the resident shard a scan runs on: the quantized column (staged from the shadow table on first use) or the raw column */
static int resident_index(scan_vtab *vt, vcolumn *v, const char *tbl, const char *col, const char *fname, int quantized, vsb_group **out) {
    if (quantized) {
        char *name = sqlite3_mprintf("vector0_%s_%s", tbl, col);
        int exists = name && sys_exists(vt->db, name, "table");
        sqlite3_free(name);
        if (!exists)
            return vtab_error(&vt->base, "Quantization table not found for table '%s' and column '%s'. Ensure that vector_quantize() has been called before using vector_quantize_scan().", tbl, col);
        if (v->qix && !v->q_user_preloaded) {
            /* lazily staged copy = a cache of the shadow table, which the reference reads per query (:2186-2227): drop it when
             * it was staged inside a transaction (rollbacks are invisible) or another connection rewrote the chunks */
            int stale = v->q_tainted;
            if (!stale) {
                sqlite3_int64 dv = query_int64(vt->db, "PRAGMA data_version;");
                if (dv != v->q_dataver) {
                    sqlite3_int64 fp[4];
                    quant_fingerprint(vt->db, v, fp);
                    stale = memcmp(fp, v->q_fp, sizeof fp) != 0;
                    v->q_dataver = dv;
                }
            }
            if (stale) { drop_qix(v); column_load_meta(vt->db, v); }
        }
        if (!v->qix) { /* not preloaded: the reference streams the chunks from disk per query (:2186-2227); we stage them once */
            char *err = 0;
            if (stage_quantized(vt->db, v, &err) != SQLITE_OK) {
                int rc = vtab_error(&vt->base, "%s: %s", fname, err ? err : "device staging failed");
                sqlite3_free(err);
                return rc;
            }
        }
        *out = v->qix;
        return SQLITE_OK;
    }
    int rc = stage_full_column(vt, v);
    if (rc != SQLITE_OK) return rc;
    *out = v->fix;
    return SQLITE_OK;
}

/* ------------------------------------------------------------------------------------------------ arguments */
static int arg_kind(const module_def *m, int i) {
    if (i < 2) return ARG_TEXT;
    if (i == 2) return ARG_VECTOR;
    if (i == 3) return m->op == OP_STREAM ? ARG_NONE : m->op == OP_RANGE ? ARG_RADIUS : ARG_K;
    return m->hidden[i - 4];
}
static int check_multiple(scan_vtab *vt, const char *fname, sqlite3_value *a, const char *what, int multiple, const char *unit) {
    if (sqlite3_value_bytes(a) % multiple == 0) return SQLITE_OK;
    return vtab_error(&vt->base, "%s: %s has %d bytes, expected a multiple of %d (%s).", fname, what, sqlite3_value_bytes(a), multiple, unit);
}
/* every check of argument i that needs no other argument: its SQL type, a BLOB's size, a count's range */
static int check_arg(scan_vtab *vt, const char *fname, int kind, int i, sqlite3_value *a) {
#define T(t) (1 << SQLITE_##t)
    static const struct { int types; const char *names; } accepts[] = {
        [ARG_TEXT] = {T(TEXT), "TEXT"},          [ARG_VECTOR] = {T(TEXT) | T(BLOB), "TEXT or BLOB"},
        [ARG_K] = {T(INTEGER), "INTEGER"},       [ARG_RADIUS] = {T(INTEGER) | T(FLOAT), "INTEGER or FLOAT"},
        [ARG_ROWIDS] = {T(BLOB), "BLOB"},        [ARG_SETS] = {T(BLOB), "BLOB"},
        [ARG_QUERY_SETS] = {T(BLOB) | T(NULL), "BLOB or NULL"}, [ARG_GROUPS] = {T(BLOB), "BLOB"},
        [ARG_LIMIT] = {T(INTEGER) | T(NULL), "INTEGER or NULL"}, [ARG_CANDIDATES] = {T(INTEGER), "INTEGER"},
    };
#undef T
    const int t = sqlite3_value_type(a);
    if (!(accepts[kind].types & (1 << t)))
        return vtab_error(&vt->base, "%s: argument %d must be of type %s (got %s).", fname, i + 1, accepts[kind].names, sql_type_name(t));
    switch (kind) {
    case ARG_K:
        if (sqlite3_value_int(a) < 0) return vtab_error(&vt->base, "%s: k must not be negative.", fname);
        break;
    case ARG_LIMIT:
        if (t == SQLITE_INTEGER && sqlite3_value_int64(a) < 0) return vtab_error(&vt->base, "%s: limit must not be negative.", fname);
        break;
    case ARG_CANDIDATES:
        if (sqlite3_value_int64(a) < 0 || sqlite3_value_int64(a) > INT32_MAX)
            return vtab_error(&vt->base, "%s: candidates must be between 0 and %d.", fname, INT32_MAX);
        break;
    case ARG_ROWIDS: return check_multiple(vt, fname, a, "rowids", 8, "int64 rowids");
    case ARG_SETS: return check_multiple(vt, fname, a, "sets", 16, "int64 set, int64 rowid pairs");
    case ARG_QUERY_SETS: return t == SQLITE_NULL ? SQLITE_OK : check_multiple(vt, fname, a, "query_sets", 8, "int64 set indexes");
    case ARG_GROUPS: return check_multiple(vt, fname, a, "groups", 16, "int64 key, int64 rowid pairs");
    }
    return SQLITE_OK;
}

/* an xFilter call once its arguments have passed: the column, its resident copy and the queries */
typedef struct {
    vcolumn *v;
    vsb_group *ix;                 /* the resident column of the module (rerank: the quantized one) */
    const uint8_t *raw;            /* nq queries of the column's type */
    const void *query;             /* the queries ix is scanned with: raw, or quantized for the quantized column */
    int nq, k;
    void *owned;                   /* queries decoded from JSON */
    uint8_t *qq;                   /* quantized queries */
} scan_call;

/* the checks of a call in one order for every module: the argument count, each argument on its own in position order, the
 * context, the queries against the column, query_sets against the queries, then the quantization table and staging
 * (resident_index); then every query is quantized for a quantized column.  The caller frees owned and qq whatever this returns. */
static int parse_call(scan_vtab *vt, const module_def *m, int argc, sqlite3_value **argv, scan_call *q) {
    const char *fname = m->name;
    memset(q, 0, sizeof *q);
    const int nargs = m->op == OP_STREAM ? 3 : 4 + nhidden(m);
    if (argc != nargs) return vtab_error(&vt->base, "%s expects %d arguments, but %d were provided.", fname, nargs, argc);
    for (int i = 0; i < argc; ++i) {
        int rc = check_arg(vt, fname, arg_kind(m, i), i, argv[i]);
        if (rc != SQLITE_OK) return rc;
    }
    const char *tbl = (const char *)sqlite3_value_text(argv[0]);
    const char *col = (const char *)sqlite3_value_text(argv[1]);
    vcolumn *v = q->v = ctx_find(vt->ctx, tbl, col);
    if (!v) return vtab_error(&vt->base, "%s: unable to retrieve context.", fname);

    const int need = v->dim * elem_size(v->vtype);
    int bytes = 0;
    if (sqlite3_value_type(argv[2]) == SQLITE_TEXT) {
        q->owned = json_to_blob(0, &vt->base, v->vtype, (const char *)sqlite3_value_text(argv[2]), &bytes, m->many ? 0 : v->dim);
        if (!q->owned) return SQLITE_ERROR;
        q->raw = (const uint8_t *)q->owned;
    } else {
        q->raw = (const uint8_t *)sqlite3_value_blob(argv[2]);
        bytes = sqlite3_value_bytes(argv[2]);
        if (!q->raw) return vtab_error(&vt->base, "%s: input vector%s cannot be NULL.", fname, m->many ? "s" : "");
        /* the reference never checks the BLOB length (SURVEY B.7) and reads out of bounds; we refuse */
        if (!m->many && bytes < need) return vtab_error(&vt->base, "%s: input vector has %d bytes, expected %d.", fname, bytes, need);
    }
    if (m->many && (bytes <= 0 || bytes % need != 0))
        return vtab_error(&vt->base, "%s: input has %d bytes, expected a positive multiple of %d (dimension %d).", fname, bytes, need, v->dim);
    const int nq = q->nq = m->many ? bytes / need : 1;
    if (m->op == OP_SETS && sqlite3_value_type(argv[5]) == SQLITE_BLOB && sqlite3_value_bytes(argv[5]) / 8 != nq)
        return vtab_error(&vt->base, "%s: query_sets holds %d set indexes for %d queries.", fname, sqlite3_value_bytes(argv[5]) / 8, nq);

    int rc = resident_index(vt, v, tbl, col, fname, m->quantized, &q->ix);
    if (rc != SQLITE_OK) return rc;
    q->query = q->raw;
    if (m->quantized) {                                                  /* quantize every query like vQuantRun does for one (:2162-2177) */
        q->qq = (uint8_t *)sqlite3_malloc64((sqlite3_uint64)nq * (sqlite3_uint64)v->dim);
        if (!q->qq) return SQLITE_NOMEM;
        for (int b = 0; b < nq; ++b) quantize_vec(v->vtype, q->raw + (size_t)b * need, q->qq + (size_t)b * v->dim, v->offset, v->scale, v->dim, v->qtype);
        q->query = q->qq;
    }
    q->k = arg_kind(m, 3) == ARG_K ? sqlite3_value_int(argv[3]) : 0;
    return SQLITE_OK;
}

/* the rows of the resident column ix whose rowid is in the (checked) rowids BLOB, as the row bitmap of the scan (sqlite3_free it) */
static int rowids_bitmap(scan_vtab *vt, const char *fname, sqlite3_value *arg, vsb_group *ix, uint32_t **out) {
    const sqlite3_int64 n = sqlite3_value_bytes(arg) / 8, rows = vsb_group_rows(ix);
    int64_t *ids = (int64_t *)sqlite3_malloc64((sqlite3_uint64)(n > 0 ? n : 1) * sizeof(int64_t));
    uint32_t *bits = (uint32_t *)sqlite3_malloc64((sqlite3_uint64)((rows + 31) / 32 + 1) * sizeof(uint32_t));
    int rc = (ids && bits) ? SQLITE_OK : SQLITE_NOMEM;
    if (rc == SQLITE_OK && n > 0) memcpy(ids, sqlite3_value_blob(arg), (size_t)n * sizeof(int64_t));   /* little-endian host */
    if (rc == SQLITE_OK && vsb_group_rowid_bitmap(ix, ids, n, bits) < 0) rc = vtab_error(&vt->base, "%s: %s", fname, vsb_last_error());
    sqlite3_free(ids);
    if (rc != SQLITE_OK) { sqlite3_free(bits); return rc; }
    *out = bits;
    return SQLITE_OK;
}

static int cmp_i64(const void *a, const void *b) {
    const int64_t x = *(const int64_t *)a, y = *(const int64_t *)b;
    return x < y ? -1 : x > y;
}

/* the (int64 key, int64 rowid) pairs of a (checked) sets / groups BLOB by key: its nkeys distinct keys ascending, key i's rowids at
 * [offsets[i], offsets[i + 1]) of rowids (pair_runs_free) */
typedef struct {
    int64_t *keys, *offsets, *rowids;
    sqlite3_int64 nkeys;
} pair_runs;
static void pair_runs_free(pair_runs *r) { sqlite3_free(r->keys); sqlite3_free(r->offsets); sqlite3_free(r->rowids); }
static int pairs_by_key(sqlite3_value *arg, pair_runs *r) {
    const sqlite3_int64 npairs = sqlite3_value_bytes(arg) / 16;
    const sqlite3_uint64 room = (sqlite3_uint64)(npairs > 0 ? npairs : 1);
    int64_t *pairs = (int64_t *)sqlite3_malloc64(room * 16);
    r->keys = (int64_t *)sqlite3_malloc64(room * sizeof(int64_t));
    r->offsets = (int64_t *)sqlite3_malloc64((room + 1) * sizeof(int64_t));
    r->rowids = (int64_t *)sqlite3_malloc64(room * sizeof(int64_t));
    r->nkeys = 0;
    const int rc = (pairs && r->keys && r->offsets && r->rowids) ? SQLITE_OK : SQLITE_NOMEM;
    if (rc == SQLITE_OK) {
        if (npairs > 0) memcpy(pairs, sqlite3_value_blob(arg), (size_t)npairs * 16);   /* little-endian host */
        qsort(pairs, (size_t)npairs, 16, cmp_i64);                                     /* by key, a pair's first int64 */
        for (sqlite3_int64 i = 0; i < npairs; ++i) {
            if (r->nkeys == 0 || r->keys[r->nkeys - 1] != pairs[2 * i]) {
                r->offsets[r->nkeys] = i;
                r->keys[r->nkeys++] = pairs[2 * i];
            }
            r->rowids[i] = pairs[2 * i + 1];
        }
        r->offsets[r->nkeys] = npairs;
    }
    sqlite3_free(pairs);
    return rc;
}

/* the sets the nq queries name, as dense bitmaps over the resident column ix (*bits: nsets x (rows + 31) / 32 words) and each
 * query's dense set index (*soq); a named set without pairs is empty and pairs of unnamed sets are skipped; sqlite3_free both */
static int sets_bitmaps(scan_vtab *vt, const char *fname, sqlite3_value *sets, sqlite3_value *qsets, int nq, vsb_group *ix,
                        uint32_t **bits, int32_t **soq, int *nsets) {
    const sqlite3_int64 words = (vsb_group_rows(ix) + 31) / 32;
    pair_runs r;
    int64_t *q = (int64_t *)sqlite3_malloc64((sqlite3_uint64)nq * sizeof(int64_t));
    int64_t *keys = (int64_t *)sqlite3_malloc64((sqlite3_uint64)nq * sizeof(int64_t));
    int32_t *dense = (int32_t *)sqlite3_malloc64((sqlite3_uint64)nq * sizeof(int32_t));
    uint32_t *out = 0;
    int rc = pairs_by_key(sets, &r), n = 0;
    if (rc == SQLITE_OK && !(q && keys && dense)) rc = SQLITE_NOMEM;
    if (rc != SQLITE_OK) goto done;
    for (int b = 0; b < nq; ++b) q[b] = sqlite3_value_type(qsets) == SQLITE_NULL ? b : ((const int64_t *)sqlite3_value_blob(qsets))[b];
    memcpy(keys, q, (size_t)nq * sizeof(int64_t));
    qsort(keys, (size_t)nq, sizeof(int64_t), cmp_i64);
    for (int b = 0; b < nq; ++b) if (n == 0 || keys[n - 1] != keys[b]) keys[n++] = keys[b];     /* distinct set indexes -> dense 0 .. n-1 */
    for (int b = 0; b < nq; ++b) dense[b] = (int32_t)((const int64_t *)bsearch(&q[b], keys, (size_t)n, sizeof(int64_t), cmp_i64) - keys);
    out = (uint32_t *)sqlite3_malloc64((sqlite3_uint64)(n > 0 ? n : 1) * (sqlite3_uint64)(words + 1) * sizeof(uint32_t));
    if (!out) { rc = SQLITE_NOMEM; goto done; }
    for (int d = 0; d < n; ++d) {
        const int64_t *run = (const int64_t *)bsearch(&keys[d], r.keys, (size_t)r.nkeys, sizeof(int64_t), cmp_i64);
        const sqlite3_int64 i = run ? run - r.keys : 0, m = run ? r.offsets[i + 1] - r.offsets[i] : 0;
        if (vsb_group_rowid_bitmap(ix, r.rowids + (run ? r.offsets[i] : 0), m, out + d * words) < 0) {
            rc = vtab_error(&vt->base, "%s: %s", fname, vsb_last_error());
            goto done;
        }
    }
done:
    pair_runs_free(&r);
    sqlite3_free(q); sqlite3_free(keys);
    if (rc != SQLITE_OK) { sqlite3_free(out); sqlite3_free(dense); return rc; }
    *bits = out; *soq = dense; *nsets = n;
    return SQLITE_OK;
}

/* ------------------------------------------------------------------------------------------------ xFilter */
static int vt_filter(sqlite3_vtab_cursor *cur, int idxnum, const char *idxstr, int argc, sqlite3_value **argv) {
    (void)idxnum; (void)idxstr;
    scan_cursor *c = (scan_cursor *)cur;
    scan_vtab *vt = (scan_vtab *)cur->pVtab;
    const module_def *m = vt->def;
    const char *fname = m->name;
    c->ngroups = 0; c->g = 0; c->j = 0;
    scan_call q;
    int rc = parse_call(vt, m, argc, argv, &q), src = VSB_OK, nsets = 0;
    sqlite3_int64 ngroups = 1;
    uint32_t *allow = 0, *setbits = 0;
    int32_t *soq = 0;
    int *counts = 0;                                                     /* rows of each query, as the top-k calls return them */
    int64_t *qids = 0, *offsets = 0;
    double *qdist = 0;
    pair_runs runs = {0};
    vsb_range *range = 0;
    vsb_grouped *res = 0;
    if (rc != SQLITE_OK) goto out;
    const int nq = q.nq, k = q.k, metric = q.v->metric;
    if (arg_kind(m, 3) == ARG_K) {
        if (k == 0) { rc = leads_group(m) ? SQLITE_OK : SQLITE_DONE; goto out; }   /* :1795-1796; the many-query and grouped modules: no rows */
        if (m->op != OP_GROUPED) {                                      /* nq groups of up to k rows */
            counts = (int *)sqlite3_malloc64((sqlite3_uint64)nq * sizeof(int));
            if ((rc = counts ? cursor_alloc(c, nq, k, m->op) : SQLITE_NOMEM) != SQLITE_OK) goto out;
            ngroups = nq;
        }
    }
    if (m->hidden[0] == ARG_ROWIDS && (rc = rowids_bitmap(vt, fname, argv[4], q.ix, &allow)) != SQLITE_OK) goto out;
    int *max_index = m->many ? 0 : &c->max_index;

    switch (m->op) {
    case OP_TOPK:
        src = allow ? vsb_group_scan_topk_filtered(q.ix, metric, q.query, nq, k, allow, vsb_group_rows(q.ix), c->ids, c->dist, counts, max_index)
                    : vsb_group_scan_topk(q.ix, metric, q.query, nq, k, c->ids, c->dist, counts, max_index);
        break;
    case OP_STREAM: {
        const sqlite3_int64 n = vsb_group_rows(q.ix);
        if ((rc = cursor_alloc(c, 1, n, m->op)) != SQLITE_OK) goto out;
        if (n > 0) src = vsb_group_scan_all(q.ix, metric, q.query, c->fdist, c->ids);
        c->count[0] = n;
        c->j = -1;
        break;
    }
    case OP_RANGE: {
        const double radius = sqlite3_value_double(argv[3]);
        src = vsb_group_scan_range(q.ix, metric, q.query, 1, &radius, allow, allow ? vsb_group_rows(q.ix) : 0, &range);
        if (src != VSB_OK) break;
        const int64_t *ids = 0;
        const double *dist = 0;
        int64_t n = 0;
        vsb_range_get(range, 0, &ids, &dist, &n);
        if ((rc = cursor_alloc(c, 1, n, m->op)) != SQLITE_OK) goto out;
        if (n > 0) {
            memcpy(c->ids, ids, (size_t)n * sizeof(int64_t));
            memcpy(c->dist, dist, (size_t)n * sizeof(double));
        }
        c->count[0] = n;
        break;
    }
    case OP_SETS:
        if ((rc = sets_bitmaps(vt, fname, argv[4], argv[5], nq, q.ix, &setbits, &soq, &nsets)) != SQLITE_OK) goto out;
        src = vsb_group_scan_topk_sets(q.ix, metric, q.query, nq, k, setbits, nsets, vsb_group_rows(q.ix), soq, c->ids, c->dist, counts, 0);
        break;
    case OP_GROUPED: {
        const sqlite3_int64 lim64 = sqlite3_value_type(argv[5]) == SQLITE_NULL ? 0 : sqlite3_value_int64(argv[5]);
        const int limit = lim64 > 0x7FFFFFFF ? 0 : (int)lim64;         /* a limit above every possible key count keeps every key */
        kept_grouping *kept = q.ix == q.v->qix ? &q.v->q_kept : &q.v->fix_kept;
        const void *blob = sqlite3_value_blob(argv[4]);
        const sqlite3_int64 bytes = sqlite3_value_bytes(argv[4]);
        if (!kept->gr || kept->bytes != bytes || (bytes > 0 && memcmp(kept->blob, blob, (size_t)bytes) != 0)) {
            /* not the kept statement's groups: lay them out anew, in place of the kept grouping */
            kept_free(kept);
            if ((rc = pairs_by_key(argv[4], &runs)) != SQLITE_OK) goto out;
            vsb_grouping *gr = 0;
            if ((src = vsb_group_grouping_create(q.ix, runs.rowids, runs.offsets, (int)runs.nkeys, &gr)) != VSB_OK) break;
            kept->blob = (unsigned char *)sqlite3_malloc64((sqlite3_uint64)(bytes > 0 ? bytes : 1));
            if (!kept->blob) { vsb_grouping_free(gr); rc = SQLITE_NOMEM; goto out; }
            if (bytes > 0) memcpy(kept->blob, blob, (size_t)bytes);
            kept->bytes = bytes;
            kept->gr = gr;
            kept->keys = runs.keys;                                     /* dense key index -> user key */
            runs.keys = 0;
        }
        src = vsb_scan_topk_grouping(kept->gr, metric, q.query, nq, k, limit, &res);
        if (src != VSB_OK) break;
        sqlite3_int64 total = 0;                                        /* every query's keys, one group each */
        for (int b = 0; b < nq; ++b) {
            int nk = 0;
            const int32_t *gk = 0;
            const int64_t *go = 0, *gi = 0;
            const double *gd = 0;
            vsb_grouped_get(res, b, &nk, &gk, &go, &gi, &gd);
            total += nk;
        }
        if ((rc = cursor_alloc(c, total, k, m->op)) != SQLITE_OK) goto out;
        sqlite3_int64 i = 0;
        for (int b = 0; b < nq; ++b) {
            int nk = 0;
            const int32_t *gk = 0;
            const int64_t *go = 0, *gi = 0;
            const double *gd = 0;
            vsb_grouped_get(res, b, &nk, &gk, &go, &gi, &gd);
            for (int t = 0; t < nk; ++t, ++i) {
                const sqlite3_int64 n = go[t + 1] - go[t];
                c->count[i] = n;
                c->key[i] = kept->keys[gk[t]];
                c->query[i] = b;
                memcpy(c->ids + (size_t)i * k, gi + go[t], (size_t)n * sizeof(int64_t));
                memcpy(c->dist + (size_t)i * k, gd + go[t], (size_t)n * sizeof(double));
            }
        }
        ngroups = total;
        break;
    }
    case OP_RERANK: {
        const int cand = (int)sqlite3_value_int64(argv[4]);
        vsb_group *fix = 0;
        /* 1: the top `candidates` of the quantized column, every query from a fresh cursor, as the subquery of the composed
         * statement; counts holds each query's candidate count until step 2 */
        offsets = (int64_t *)sqlite3_malloc64((sqlite3_uint64)(nq + 1) * sizeof(int64_t));
        qids = (int64_t *)sqlite3_malloc64((sqlite3_uint64)nq * (sqlite3_uint64)(cand > 0 ? cand : 1) * sizeof(int64_t));
        qdist = (double *)sqlite3_malloc64((sqlite3_uint64)nq * (sqlite3_uint64)(cand > 0 ? cand : 1) * sizeof(double));
        if (!offsets || !qids || !qdist) { rc = SQLITE_NOMEM; goto out; }
        memset(counts, 0, (size_t)nq * sizeof(int));
        int fresh = 0;
        if (cand > 0 && (src = vsb_group_scan_topk(q.ix, metric, q.query, nq, cand, qids, qdist, counts, &fresh)) != VSB_OK) break;
        offsets[0] = 0;                                                  /* each query's candidate rowids, back to back */
        for (int b = 0; b < nq; ++b) {
            memmove(qids + offsets[b], qids + (size_t)b * (size_t)cand, (size_t)counts[b] * sizeof(int64_t));
            offsets[b + 1] = offsets[b] + counts[b];
        }
        /* 2: the rerank on the raw column, reading only the candidate rows */
        if ((rc = resident_index(vt, q.v, (const char *)sqlite3_value_text(argv[0]), (const char *)sqlite3_value_text(argv[1]), fname, 0, &fix)) != SQLITE_OK)
            goto out;
        src = vsb_group_scan_topk_rows(fix, metric, q.raw, nq, k, qids, offsets, c->ids, c->dist, counts, max_index);
        break;
    }
    }
    if (src != VSB_OK) { rc = vtab_error(&vt->base, "%s: %s", fname, vsb_last_error()); goto out; }
    if (counts) for (int b = 0; b < nq; ++b) c->count[b] = counts[b];
    c->ngroups = ngroups;
    skip_empty(c);
out:
    sqlite3_free(q.owned); sqlite3_free(q.qq);
    sqlite3_free(allow); sqlite3_free(setbits); sqlite3_free(soq); sqlite3_free(counts);
    sqlite3_free(qids); sqlite3_free(qdist); sqlite3_free(offsets);
    pair_runs_free(&runs);
    vsb_range_free(range);
    vsb_grouped_free(res);
    return rc;
}

static const sqlite3_module scan_module = {0, 0, vt_connect, vt_best_index, vt_disconnect, 0, vt_open, vt_close, vt_filter, vt_next,
                                           vt_eof, vt_column, vt_rowid, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};

/* vector_rowid_set(x): aggregate of the non-NULL x as the rowids BLOB of the *_filtered modules (int64, host byte order =
 * little-endian), e.g. (SELECT vector_rowid_set(rowid) FROM docs WHERE lang = 'en'); no rows give an empty BLOB */
typedef struct {
    int64_t *v;
    sqlite3_int64 n, cap;
} rowid_set;
static void rowid_set_step(sqlite3_context *ctx, int argc, sqlite3_value **argv) {
    (void)argc;
    if (sqlite3_value_type(argv[0]) == SQLITE_NULL) return;
    rowid_set *s = (rowid_set *)sqlite3_aggregate_context(ctx, (int)sizeof *s);
    if (!s) { sqlite3_result_error_code(ctx, SQLITE_NOMEM); return; }
    if (s->n == s->cap) {
        const sqlite3_int64 cap = s->cap ? 2 * s->cap : 1024;
        int64_t *v = (int64_t *)sqlite3_malloc64((sqlite3_uint64)cap * sizeof(int64_t));
        if (!v) { sqlite3_result_error_code(ctx, SQLITE_NOMEM); return; }
        if (s->n) memcpy(v, s->v, (size_t)s->n * sizeof(int64_t));
        sqlite3_free(s->v);
        s->v = v;
        s->cap = cap;
    }
    s->v[s->n++] = (int64_t)sqlite3_value_int64(argv[0]);
}
static void rowid_set_emit(sqlite3_context *ctx, const char *fname, const char *what) {
    rowid_set *s = (rowid_set *)sqlite3_aggregate_context(ctx, 0);
    if (!s || s->n == 0) {
        sqlite3_result_blob(ctx, "", 0, SQLITE_STATIC);
    } else if (s->n > INT32_MAX / 8) {
        fn_error(ctx, SQLITE_ERROR,"%s: %lld %s do not fit in one BLOB.", fname, (long long)s->n, what);
    } else {
        sqlite3_result_blob(ctx, s->v, (int)(s->n * 8), SQLITE_TRANSIENT);
    }
    if (s) sqlite3_free(s->v);
}
static void rowid_set_final(sqlite3_context *ctx) { rowid_set_emit(ctx, "vector_rowid_set", "rowids"); }

/* vector_rowid_sets(set, rowid): aggregate of the rows where neither is NULL as the `sets` BLOB of vector_*_scan_batch_sets:
 * little-endian (int64 set, int64 rowid) pairs, e.g. (SELECT vector_rowid_sets(tenant, rowid) FROM docs) */
static void rowid_sets_step(sqlite3_context *ctx, int argc, sqlite3_value **argv) {
    (void)argc;
    if (sqlite3_value_type(argv[0]) == SQLITE_NULL || sqlite3_value_type(argv[1]) == SQLITE_NULL) return;
    rowid_set_step(ctx, 1, argv);
    rowid_set *s = (rowid_set *)sqlite3_aggregate_context(ctx, 0);
    if (s && s->n % 2 == 1) rowid_set_step(ctx, 1, argv + 1);         /* the set was appended: now its rowid */
}
static void rowid_sets_final(sqlite3_context *ctx) { rowid_set_emit(ctx, "vector_rowid_sets", "values"); }

/* ------------------------------------------------------------------------------------------------ entry point */
__attribute__((visibility("default"))) int sqlite3_vector_init(sqlite3 *db, char **err, const sqlite3_api_routines *api) { /* :2555-2638 */
    vsq_api = api;
    int rc = sqlite3_exec(db, "CREATE TABLE IF NOT EXISTS _sqliteai_vector (tblname TEXT, colname TEXT, key TEXT, value ANY, PRIMARY KEY(tblname, colname, key));", 0, 0, 0);
    if (rc != SQLITE_OK) return rc;
    vcontext *ctx = (vcontext *)sqlite3_malloc((int)sizeof *ctx);
    if (!ctx) {
        if (err) *err = sqlite3_mprintf("Out of memory: failed to allocate vector extension context.");
        return SQLITE_NOMEM;
    }
    memset(ctx, 0, sizeof *ctx);
    rc = sqlite3_create_function_v2(db, "vector_version", 0, SQLITE_UTF8, ctx, fn_version, 0, 0, ctx_free); /* owns ctx */
    if (rc != SQLITE_OK) return rc;
    struct { const char *name; int nargs; void (*fn)(sqlite3_context *, int, sqlite3_value **); } fns[] = {
        {"vector_backend", 0, fn_backend},      {"vector_init", 3, fn_init},
        {"vector_quantize", 3, fn_quantize3},   {"vector_quantize", 2, fn_quantize2},
        {"vector_quantize_memory", 2, fn_quantize_memory}, {"vector_quantize_preload", 2, fn_quantize_preload},
        {"vector_quantize_cleanup", 2, fn_quantize_cleanup},
        {"vector_as_f32", 1, fn_as_f32}, {"vector_as_f32", 2, fn_as_f32}, {"vector_as_f16", 1, fn_as_f16}, {"vector_as_f16", 2, fn_as_f16},
        {"vector_as_bf16", 1, fn_as_bf16}, {"vector_as_bf16", 2, fn_as_bf16}, {"vector_as_i8", 1, fn_as_i8}, {"vector_as_i8", 2, fn_as_i8},
        {"vector_as_u8", 1, fn_as_u8}, {"vector_as_u8", 2, fn_as_u8},
    };
    for (size_t i = 0; i < sizeof fns / sizeof fns[0]; ++i) {
        rc = sqlite3_create_function(db, fns[i].name, fns[i].nargs, SQLITE_UTF8, ctx, fns[i].fn, 0, 0);
        if (rc != SQLITE_OK) return rc;
    }
    if ((rc = sqlite3_create_function(db, "vector_rowid_set", 1, SQLITE_UTF8, ctx, 0, rowid_set_step, rowid_set_final)) != SQLITE_OK) return rc;
    if ((rc = sqlite3_create_function(db, "vector_rowid_sets", 2, SQLITE_UTF8, ctx, 0, rowid_sets_step, rowid_sets_final)) != SQLITE_OK) return rc;
    for (int i = 0; i < N_MODULES; ++i) {
        ctx->mods[i].def = &modules[i];
        ctx->mods[i].ctx = ctx;
        if ((rc = sqlite3_create_module(db, modules[i].name, &scan_module, &ctx->mods[i])) != SQLITE_OK) return rc;
    }
    return SQLITE_OK;
}
