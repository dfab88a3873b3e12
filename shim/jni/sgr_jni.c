/* sgr_jni.c — JNI glue between surge.gpu.Native (shim/scala) and include/sgr.h.
 * Built only where a JDK exists (needs <jni.h>):  gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux
 *     -I../../include sgr_jni.c -L../../surge_b200/lib -lsgr -o libsgr_jni.so
 * The build image of this repository has no JDK, so this file is guarded and compiled nowhere here; all logic lives
 * behind the C ABI, which the Python/ctypes tests cover. */
#if defined(__has_include)
#if __has_include(<jni.h>)
#include <jni.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "sgr.h"

#define H(h) ((sgr_engine*)(intptr_t)(h))

/* Lengths and buffers come from Java: check them here, throw IllegalArgumentException, never read past what was handed over
 * (round-1 review: a short `firsts` array, a non-direct buffer (GetDirectBufferAddress == NULL) or an nbytes beyond the
 * buffer's capacity went straight to the C ABI). */
static int bad_arg(JNIEnv* env, const char* what) {
  (*env)->ThrowNew(env, (*env)->FindClass(env, "java/lang/IllegalArgumentException"), what);
  return SGR_ERR_INVALID;
}
/* direct buffer address, checked: non-NULL and at least `need` bytes of capacity */
static void* direct(JNIEnv* env, jobject buf, jlong need, const char* what, int* ok) {
  void* p = buf ? (*env)->GetDirectBufferAddress(env, buf) : 0;
  if (!p || need < 0 || (*env)->GetDirectBufferCapacity(env, buf) < need) { bad_arg(env, what); *ok = 0; return 0; }
  return p;
}

static void throw_for(JNIEnv* env, sgr_engine* e, int32_t rc) {
  const char* cls = rc == SGR_ERR_STATE ? "org/apache/kafka/streams/errors/InvalidStateStoreException" : "java/lang/RuntimeException";
  (*env)->ThrowNew(env, (*env)->FindClass(env, cls), sgr_last_error(e));
}

JNIEXPORT jlong JNICALL Java_surge_gpu_Native_00024_create(JNIEnv* env, jobject o, jint device) {
  sgr_config cfg; memset(&cfg, 0, sizeof cfg); cfg.device = device;
  sgr_engine* e = 0;
  int32_t rc = sgr_create(&cfg, &e);
  if (rc != SGR_OK) { throw_for(env, 0, rc); return 0; }  /* SGR_ERR_NO_DEVICE: fail loudly, never fall back */
  return (jlong)(intptr_t)e;
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_destroy(JNIEnv* env, jobject o, jlong h) { return sgr_destroy(H(h)); }
JNIEXPORT jstring JNICALL Java_surge_gpu_Native_00024_lastError(JNIEnv* env, jobject o, jlong h) { return (*env)->NewStringUTF(env, sgr_last_error(H(h))); }
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_registerProgram(JNIEnv* env, jobject o, jlong h, jobject prog) {
  int ok = 1; void* p = direct(env, prog, (jlong)sizeof(sgr_fold_program), "program: direct buffer of sizeof(sgr_fold_program) bytes", &ok);
  return ok ? sgr_register_program(H(h), (const sgr_fold_program*)p) : SGR_ERR_INVALID;
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_loadEvents(JNIEnv* env, jobject o, jlong h, jobject ev, jlong nbytes, jobject offs, jlong n_agg) {
  int ok = 1;
  void* e = direct(env, ev, nbytes, "events: direct buffer shorter than nbytes", &ok);
  void* so = ok && n_agg >= 0 ? direct(env, offs, (n_agg + 1) * 8, "segOffsets: direct buffer of (nAgg + 1) u64", &ok) : 0;
  return ok && so ? sgr_load_events(H(h), e, (uint64_t)nbytes, (const uint64_t*)so, (uint64_t)n_agg) : SGR_ERR_INVALID;
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_loadUnsorted(JNIEnv* env, jobject o, jlong h, jobject rec, jlong n, jlong n_agg) {
  int ok = 1; void* r = n >= 0 && n <= (INT64_MAX / 64) ? direct(env, rec, n * 64, "records: direct buffer shorter than nRecords * 64", &ok) : (bad_arg(env, "nRecords"), (void*)0);
  return ok && r ? sgr_load_unsorted(H(h), r, (uint64_t)n, (uint64_t)n_agg) : SGR_ERR_INVALID;
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_setInitialStates(JNIEnv* env, jobject o, jlong h, jobject st, jlong n_agg) {
  if (!st) return sgr_set_initial_states(H(h), 0, 0);
  int ok = 1; void* p = direct(env, st, 16 * n_agg, "states: direct buffer shorter than nAgg states", &ok);   /* >= 16 bytes per state */
  return ok ? sgr_set_initial_states(H(h), p, (uint64_t)n_agg) : SGR_ERR_INVALID;
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_fold(JNIEnv* env, jobject o, jlong h) { return sgr_fold(H(h)); }
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_foldIncremental(JNIEnv* env, jobject o, jlong h, jobject rec, jlong n) {
  int ok = 1; void* r = n >= 0 && n <= (INT64_MAX / 64) ? direct(env, rec, n * 64, "records: direct buffer shorter than nRecords * 64", &ok) : (bad_arg(env, "nRecords"), (void*)0);
  return ok && r ? sgr_fold_incremental(H(h), r, (uint64_t)n) : SGR_ERR_INVALID;
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_loadKeys(JNIEnv* env, jobject o, jlong h, jobject keys, jobject offs, jlong n) {
  int ok = 1;
  const uint32_t* ko = n >= 0 ? (const uint32_t*)direct(env, offs, (n + 1) * 4, "keyOffsets: direct buffer of (n + 1) u32", &ok) : 0;
  if (!ok || !ko) return SGR_ERR_INVALID;
  const uint8_t* k = (const uint8_t*)direct(env, keys, (jlong)ko[n], "keys: direct buffer shorter than keyOffsets[n]", &ok);
  return ok ? sgr_load_keys(H(h), k, ko, (uint64_t)n) : SGR_ERR_INVALID;
}
JNIEXPORT jbyteArray JNICALL Java_surge_gpu_Native_00024_get(JNIEnv* env, jobject o, jlong h, jbyteArray key) {
  jsize klen = (*env)->GetArrayLength(env, key);
  jbyte* k = (*env)->GetByteArrayElements(env, key, 0);
  uint8_t out[SGR_MAX_STATE_BYTES]; uint32_t outlen = 0; int32_t exists = 0;
  int32_t rc = sgr_get(H(h), (const uint8_t*)k, (uint32_t)klen, out, sizeof out, &outlen, &exists);
  (*env)->ReleaseByteArrayElements(env, key, k, JNI_ABORT);
  if (rc != SGR_OK) { throw_for(env, H(h), rc); return 0; }
  if (!exists) return 0;                                   /* Option.empty */
  jbyteArray r = (*env)->NewByteArray(env, (jsize)outlen);  /* a fresh array, as RocksDB returns */
  (*env)->SetByteArrayRegion(env, r, 0, (jsize)outlen, (const jbyte*)out);
  return r;
}
/* out and flags are direct buffers of n rows of (state_bytes - 8) bytes and n u32; SGR_ERR_CAPACITY when out is too short */
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_getBatch(JNIEnv* env, jobject o, jlong h, jobject keys, jobject offs, jlong n, jobject out, jobject flags) {
  int ok = 1;
  const uint32_t* ko = n >= 0 ? (const uint32_t*)direct(env, offs, (n + 1) * 4, "keyOffsets: direct buffer of (n + 1) u32", &ok) : 0;
  if (!ok || !ko) return n < 0 ? bad_arg(env, "n must be non-negative") : SGR_ERR_INVALID;
  const uint8_t* k = ko[n] ? (const uint8_t*)direct(env, keys, (jlong)ko[n], "keys: direct buffer shorter than keyOffsets[n]", &ok) : 0;
  uint32_t* fl = ok ? (uint32_t*)direct(env, flags, n * 4, "flags: direct buffer of n u32", &ok) : 0;
  void* rows = ok ? direct(env, out, 0, "out: direct buffer", &ok) : 0;
  if (!ok) return SGR_ERR_INVALID;
  int32_t rc = sgr_get_batch(H(h), k, ko, (uint64_t)n, rows, (uint64_t)(*env)->GetDirectBufferCapacity(env, out), fl, 0);
  if (rc != SGR_OK) throw_for(env, H(h), rc);
  return rc;
}
/* One sgr_put_batch. keys / keyOffsets as for getBatch; rows: a direct buffer of n x (stateBytes - 8) bytes, stateBytes being
 * the registered program's (checked against the table's when there is one); present: a direct buffer of n bytes (0 = a
 * tombstone). Returns the ids appended, or -1 after throwing (InvalidStateStoreException on a key table of an ingest). */
JNIEXPORT jlong JNICALL Java_surge_gpu_Native_00024_putBatch(JNIEnv* env, jobject o, jlong h, jobject keys, jobject offs, jlong n, jobject rows,
                                                             jint state_bytes, jobject present) {
  int ok = 1;
  if (n < 0 || n > INT64_MAX / SGR_MAX_STATE_BYTES) { bad_arg(env, "n must be non-negative"); return -1; }
  if (state_bytes < 16 || state_bytes > (jint)SGR_MAX_STATE_BYTES) { bad_arg(env, "stateBytes out of range"); return -1; }
  uint32_t sb = 0;
  if (sgr_states_device(H(h), 0, 0, &sb) == SGR_OK && sb != (uint32_t)state_bytes) { bad_arg(env, "stateBytes is not the program's"); return -1; }
  const uint32_t* ko = (const uint32_t*)direct(env, offs, (n + 1) * 4, "keyOffsets: direct buffer of (n + 1) u32", &ok);
  if (!ok) return -1;
  const uint8_t* k = ko[n] ? (const uint8_t*)direct(env, keys, (jlong)ko[n], "keys: direct buffer shorter than keyOffsets[n]", &ok) : 0;
  const void* r = ok ? direct(env, rows, n * (state_bytes - 8), "rows: direct buffer of n x (stateBytes - 8) bytes", &ok) : 0;
  const uint8_t* p = ok ? (const uint8_t*)direct(env, present, n, "present: direct buffer of n bytes", &ok) : 0;
  if (!ok) return -1;
  uint64_t n_new = 0;
  int32_t rc = sgr_put_batch(H(h), k, ko, (uint64_t)n, r, p, &n_new);
  if (rc != SGR_OK) { throw_for(env, H(h), rc); return -1; }
  return (jlong)n_new;
}
/* One page of sgr_export_changes. cursor: direct buffer of 4 u64 (next, token, nKeys, reserved), read and updated in place;
 * flags / errIdx / indices / idOffsets: direct buffers of maxRows u32 / u32 / i64 / maxRows + 1 u32; rows: maxRows x
 * (state_bytes - 8) bytes; ids: a direct buffer whose capacity is the page's id-byte budget. Returns the rows written, or -1
 * after throwing (InvalidStateStoreException when the table changed since the export's first page). */
JNIEXPORT jlong JNICALL Java_surge_gpu_Native_00024_exportChanges(JNIEnv* env, jobject o, jlong h, jint select, jobject cursor, jlong max_rows,
                                                                  jobject rows, jobject flags, jobject err_idx, jobject indices, jobject ids,
                                                                  jobject id_offsets) {
  int ok = 1;
  if (max_rows <= 0 || max_rows > INT64_MAX / (8 * SGR_MAX_STATE_BYTES)) { bad_arg(env, "maxRows must be positive"); return -1; }
  uint32_t sb = 0;
  const jlong user = sgr_states_device(H(h), 0, 0, &sb) == SGR_OK ? (jlong)sb - 8 : 0;   /* (no table yet: the call below says so) */
  sgr_changes_cursor* cur = (sgr_changes_cursor*)direct(env, cursor, (jlong)sizeof(sgr_changes_cursor), "cursor: direct buffer of 4 u64", &ok);
  void* rw = ok ? direct(env, rows, max_rows * user, "rows: direct buffer shorter than maxRows states", &ok) : 0;
  uint32_t* fl = ok ? (uint32_t*)direct(env, flags, max_rows * 4, "flags: direct buffer of maxRows u32", &ok) : 0;
  uint32_t* er = ok ? (uint32_t*)direct(env, err_idx, max_rows * 4, "errIdx: direct buffer of maxRows u32", &ok) : 0;
  int64_t* ix = ok ? (int64_t*)direct(env, indices, max_rows * 8, "indices: direct buffer of maxRows i64", &ok) : 0;
  uint32_t* io = ok ? (uint32_t*)direct(env, id_offsets, (max_rows + 1) * 4, "idOffsets: direct buffer of maxRows + 1 u32", &ok) : 0;
  uint8_t* id = ok ? (uint8_t*)direct(env, ids, 1, "ids: direct buffer", &ok) : 0;
  if (!ok) return -1;
  uint64_t n = 0;
  int32_t rc = sgr_export_changes(H(h), (uint32_t)select, cur, (uint64_t)max_rows, rw, fl, er, ix, id, (uint64_t)(*env)->GetDirectBufferCapacity(env, ids),
                                  io, &n);
  if (rc != SGR_OK) { throw_for(env, H(h), rc); return -1; }
  return (jlong)n;
}
/* One page of sgr_scan. from / to: byte arrays, or null for an open end; fromExclusive leaves the id equal to from out. rows:
 * maxRows x (state_bytes - 8) bytes; flags / indices / idOffsets: direct buffers of maxRows u32 / maxRows i64 / maxRows + 1 u32;
 * ids: a direct buffer whose capacity is the page's id-byte budget. Returns 2 * (rows written) + 1 when a live row in range was
 * left out of the page (+ 0 when the scan is complete), or -1 after throwing. */
JNIEXPORT jlong JNICALL Java_surge_gpu_Native_00024_scan(JNIEnv* env, jobject o, jlong h, jbyteArray from, jboolean from_exclusive, jbyteArray to,
                                                         jlong max_rows, jobject rows, jobject flags, jobject indices, jobject ids, jobject id_offsets) {
  static const uint8_t empty = 0;
  int ok = 1;
  if (max_rows <= 0 || max_rows > INT64_MAX / (8 * SGR_MAX_STATE_BYTES)) { bad_arg(env, "maxRows must be positive"); return -1; }
  uint32_t sb = 0;
  const jlong user = sgr_states_device(H(h), 0, 0, &sb) == SGR_OK ? (jlong)sb - 8 : 0;   /* (no table yet: the call below says so) */
  void* rw = direct(env, rows, max_rows * user, "rows: direct buffer shorter than maxRows states", &ok);
  uint32_t* fl = ok ? (uint32_t*)direct(env, flags, max_rows * 4, "flags: direct buffer of maxRows u32", &ok) : 0;
  int64_t* ix = ok ? (int64_t*)direct(env, indices, max_rows * 8, "indices: direct buffer of maxRows i64", &ok) : 0;
  uint32_t* io = ok ? (uint32_t*)direct(env, id_offsets, (max_rows + 1) * 4, "idOffsets: direct buffer of maxRows + 1 u32", &ok) : 0;
  uint8_t* id = ok ? (uint8_t*)direct(env, ids, 1, "ids: direct buffer", &ok) : 0;
  if (!ok) return -1;
  const jsize from_len = from ? (*env)->GetArrayLength(env, from) : 0, to_len = to ? (*env)->GetArrayLength(env, to) : 0;
  jbyte* f = from ? (*env)->GetByteArrayElements(env, from, 0) : 0;
  jbyte* t = to ? (*env)->GetByteArrayElements(env, to, 0) : 0;
  uint64_t n = 0;
  int32_t more = 0;
  int32_t rc = sgr_scan(H(h), from ? (f ? (const uint8_t*)f : &empty) : 0, (uint32_t)from_len, from_exclusive ? 1 : 0,
                        to ? (t ? (const uint8_t*)t : &empty) : 0, (uint32_t)to_len, (uint64_t)max_rows, rw, fl, ix, id,
                        (uint64_t)(*env)->GetDirectBufferCapacity(env, ids), io, &n, &more);
  if (f) (*env)->ReleaseByteArrayElements(env, from, f, JNI_ABORT);
  if (t) (*env)->ReleaseByteArrayElements(env, to, t, JNI_ABORT);
  if (rc != SGR_OK) { throw_for(env, H(h), rc); return -1; }
  return (jlong)(2 * n + (more ? 1 : 0));
}
/* sgr_set_state_writer. table: a direct buffer of tableBytes bytes, per member (little endian) u32 kind (SGR_JSON_*), u32 program
 * byte offset, u32 PSTR slot bytes, u32 name length, then the name's UTF-8 bytes; nMembers == 0 clears the writer. */
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_setStateWriter(JNIEnv* env, jobject o, jlong h, jobject table, jlong table_bytes, jint n_members) {
  int ok = 1;
  if (n_members < 0 || n_members > 32 || table_bytes < 0) return bad_arg(env, "nMembers: 0 to 32 members");
  const uint8_t* t = n_members ? (const uint8_t*)direct(env, table, table_bytes, "table: direct buffer shorter than tableBytes", &ok) : 0;
  if (!ok) return SGR_ERR_INVALID;
  sgr_json_field f[32];
  char name_buf[32][256];
  jlong at = 0;
  for (jint i = 0; i < n_members; ++i) {
    uint32_t w[4];
    if (table_bytes - at < 16) return bad_arg(env, "table: a member runs past tableBytes");
    memcpy(w, t + at, 16);
    at += 16;
    if (w[0] > 255 || w[1] > 0xffff || w[3] > 255 || (jlong)w[3] > table_bytes - at) return bad_arg(env, "table: kind, offset or name length out of range");
    memcpy(name_buf[i], t + at, w[3]);
    name_buf[i][w[3]] = 0;
    at += w[3];
    if (strlen(name_buf[i]) != w[3]) return bad_arg(env, "table: a name holds a NUL byte");
    memset(&f[i], 0, sizeof f[i]);
    f[i].name = name_buf[i]; f[i].kind = (uint8_t)w[0]; f[i].dst_off = (uint16_t)w[1]; f[i].len = w[2];
  }
  int32_t rc = sgr_set_state_writer(H(h), f, (uint32_t)n_members);
  if (rc != SGR_OK) throw_for(env, H(h), rc);
  return rc;
}
/* sgr_set_state_writer_framing: SGR_VALUE_JSON (2) or SGR_VALUE_PROTOBUF_JSON (3, the multilanguage State around each value). */
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_setStateWriterFraming(JNIEnv* env, jobject o, jlong h, jint framing) {
  int32_t rc = sgr_set_state_writer_framing(H(h), framing);
  if (rc != SGR_OK) throw_for(env, H(h), rc);
  return rc;
}
/* One sgr_get_batch_values. keys / keyOffsets as for getBatch; values: a direct buffer whose capacity is the byte budget;
 * valueOffsets: n + 1 u64; flags: n u32. Returns the value bytes written, or -(bytes needed) when values is too small (nothing
 * written); throws on every other failure (a row the writer refuses, no writer: InvalidStateStoreException). */
JNIEXPORT jlong JNICALL Java_surge_gpu_Native_00024_getBatchValues(JNIEnv* env, jobject o, jlong h, jobject keys, jobject offs, jlong n, jobject values,
                                                                   jobject value_offsets, jobject flags) {
  int ok = 1;
  if (n < 0 || n > INT64_MAX / 16) { bad_arg(env, "n must be non-negative"); return 0; }
  const uint32_t* ko = (const uint32_t*)direct(env, offs, (n + 1) * 4, "keyOffsets: direct buffer of (n + 1) u32", &ok);
  if (!ok) return 0;
  const uint8_t* k = ko[n] ? (const uint8_t*)direct(env, keys, (jlong)ko[n], "keys: direct buffer shorter than keyOffsets[n]", &ok) : 0;
  uint64_t* vo = ok ? (uint64_t*)direct(env, value_offsets, (n + 1) * 8, "valueOffsets: direct buffer of (n + 1) u64", &ok) : 0;
  uint32_t* fl = ok ? (uint32_t*)direct(env, flags, n * 4, "flags: direct buffer of n u32", &ok) : 0;
  uint8_t* v = ok ? (uint8_t*)direct(env, values, 0, "values: direct buffer", &ok) : 0;
  if (!ok) return 0;
  uint64_t need = 0;
  int32_t rc = sgr_get_batch_values(H(h), k, ko, (uint64_t)n, v, (uint64_t)(*env)->GetDirectBufferCapacity(env, values), vo, fl, 0, &need);
  if (rc == SGR_ERR_CAPACITY) return -(jlong)need;
  if (rc != SGR_OK) { throw_for(env, H(h), rc); return 0; }
  return (jlong)need;
}
/* One page of sgr_export_changes_values: as exportChanges, with values (a direct buffer whose capacity is the page's value-byte
 * budget) and valueOffsets (maxRows + 1 u64) in place of rows. Returns the rows written, or -1 after throwing. */
JNIEXPORT jlong JNICALL Java_surge_gpu_Native_00024_exportChangesValues(JNIEnv* env, jobject o, jlong h, jint select, jobject cursor, jlong max_rows,
                                                                        jobject values, jobject value_offsets, jobject flags, jobject err_idx,
                                                                        jobject indices, jobject ids, jobject id_offsets) {
  int ok = 1;
  if (max_rows <= 0 || max_rows > INT64_MAX / 16) { bad_arg(env, "maxRows must be positive"); return -1; }
  sgr_changes_cursor* cur = (sgr_changes_cursor*)direct(env, cursor, (jlong)sizeof(sgr_changes_cursor), "cursor: direct buffer of 4 u64", &ok);
  uint8_t* v = ok ? (uint8_t*)direct(env, values, 1, "values: direct buffer", &ok) : 0;
  uint64_t* vo = ok ? (uint64_t*)direct(env, value_offsets, (max_rows + 1) * 8, "valueOffsets: direct buffer of maxRows + 1 u64", &ok) : 0;
  uint32_t* fl = ok ? (uint32_t*)direct(env, flags, max_rows * 4, "flags: direct buffer of maxRows u32", &ok) : 0;
  uint32_t* er = ok ? (uint32_t*)direct(env, err_idx, max_rows * 4, "errIdx: direct buffer of maxRows u32", &ok) : 0;
  int64_t* ix = ok ? (int64_t*)direct(env, indices, max_rows * 8, "indices: direct buffer of maxRows i64", &ok) : 0;
  uint32_t* io = ok ? (uint32_t*)direct(env, id_offsets, (max_rows + 1) * 4, "idOffsets: direct buffer of maxRows + 1 u32", &ok) : 0;
  uint8_t* id = ok ? (uint8_t*)direct(env, ids, 1, "ids: direct buffer", &ok) : 0;
  if (!ok) return -1;
  uint64_t n = 0;
  int32_t rc = sgr_export_changes_values(H(h), (uint32_t)select, cur, (uint64_t)max_rows, v, (uint64_t)(*env)->GetDirectBufferCapacity(env, values), vo,
                                         fl, er, ix, id, (uint64_t)(*env)->GetDirectBufferCapacity(env, ids), io, &n);
  if (rc != SGR_OK) { throw_for(env, H(h), rc); return -1; }
  return (jlong)n;
}
/* One page of sgr_scan_values: as scan, with values and valueOffsets (maxRows + 1 u64) in place of rows. Returns 2 * (rows
 * written) + 1 when a live row in range was left out of the page (+ 0 when the scan is complete), or -1 after throwing. */
JNIEXPORT jlong JNICALL Java_surge_gpu_Native_00024_scanValues(JNIEnv* env, jobject o, jlong h, jbyteArray from, jboolean from_exclusive, jbyteArray to,
                                                               jlong max_rows, jobject values, jobject value_offsets, jobject flags, jobject indices,
                                                               jobject ids, jobject id_offsets) {
  static const uint8_t empty = 0;
  int ok = 1;
  if (max_rows <= 0 || max_rows > INT64_MAX / 16) { bad_arg(env, "maxRows must be positive"); return -1; }
  uint8_t* v = (uint8_t*)direct(env, values, 1, "values: direct buffer", &ok);
  uint64_t* vo = ok ? (uint64_t*)direct(env, value_offsets, (max_rows + 1) * 8, "valueOffsets: direct buffer of maxRows + 1 u64", &ok) : 0;
  uint32_t* fl = ok ? (uint32_t*)direct(env, flags, max_rows * 4, "flags: direct buffer of maxRows u32", &ok) : 0;
  int64_t* ix = ok ? (int64_t*)direct(env, indices, max_rows * 8, "indices: direct buffer of maxRows i64", &ok) : 0;
  uint32_t* io = ok ? (uint32_t*)direct(env, id_offsets, (max_rows + 1) * 4, "idOffsets: direct buffer of maxRows + 1 u32", &ok) : 0;
  uint8_t* id = ok ? (uint8_t*)direct(env, ids, 1, "ids: direct buffer", &ok) : 0;
  if (!ok) return -1;
  const jsize from_len = from ? (*env)->GetArrayLength(env, from) : 0, to_len = to ? (*env)->GetArrayLength(env, to) : 0;
  jbyte* f = from ? (*env)->GetByteArrayElements(env, from, 0) : 0;
  jbyte* t = to ? (*env)->GetByteArrayElements(env, to, 0) : 0;
  uint64_t n = 0;
  int32_t more = 0;
  int32_t rc = sgr_scan_values(H(h), from ? (f ? (const uint8_t*)f : &empty) : 0, (uint32_t)from_len, from_exclusive ? 1 : 0,
                               to ? (t ? (const uint8_t*)t : &empty) : 0, (uint32_t)to_len, (uint64_t)max_rows, v,
                               (uint64_t)(*env)->GetDirectBufferCapacity(env, values), vo, fl, ix, id, (uint64_t)(*env)->GetDirectBufferCapacity(env, ids),
                               io, &n, &more);
  if (f) (*env)->ReleaseByteArrayElements(env, from, f, JNI_ABORT);
  if (t) (*env)->ReleaseByteArrayElements(env, to, t, JNI_ABORT);
  if (rc != SGR_OK) { throw_for(env, H(h), rc); return -1; }
  return (jlong)(2 * n + (more ? 1 : 0));
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_exportStates(JNIEnv* env, jobject o, jlong h, jobject out, jobject changed) {
  return sgr_export_states(H(h), (*env)->GetDirectBufferAddress(env, out), (uint64_t)(*env)->GetDirectBufferCapacity(env, out), 0,
                           changed ? (uint8_t*)(*env)->GetDirectBufferAddress(env, changed) : 0, 0);
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_partitionForKey(JNIEnv* env, jobject o, jbyteArray key, jint n, jboolean up_to_colon) {
  jsize klen = (*env)->GetArrayLength(env, key);
  jbyte* k = (*env)->GetByteArrayElements(env, key, 0);
  int32_t p = -1;
  int32_t rc = n > 0 ? sgr_partition_for_key_utf8((const uint8_t*)k, (uint32_t)klen, (uint32_t)n, up_to_colon ? 1 : 0, &p) : SGR_ERR_INVALID;
  (*env)->ReleaseByteArrayElements(env, key, k, JNI_ABORT);
  if (rc != SGR_OK) { bad_arg(env, "partitionForKey: numPartitions must be positive and the key valid UTF-8"); return -1; }
  return p;
}

/* ---- ingest (raw Kafka record batches) */
#define G(g) ((sgr_ingest*)(intptr_t)(g))
JNIEXPORT jlong JNICALL Java_surge_gpu_Native_00024_ingestCreate(JNIEnv* env, jobject o) {
  sgr_ingest* g = 0;
  if (sgr_ingest_create(&g) != SGR_OK) { (*env)->ThrowNew(env, (*env)->FindClass(env, "java/lang/OutOfMemoryError"), "sgr_ingest_create"); return 0; }
  return (jlong)(intptr_t)g;
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_ingestDestroy(JNIEnv* env, jobject o, jlong g) { return sgr_ingest_destroy(G(g)); }
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_ingestSetValueFraming(JNIEnv* env, jobject o, jlong g, jint framing) { return sgr_ingest_set_value_framing(G(g), framing); }
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_ingestSetNullValueType(JNIEnv* env, jobject o, jlong g, jint event_type) { return sgr_ingest_set_null_value_type(G(g), event_type); }
/* A JSON member table (sgr_ingest_set_json_packer, sgr_dingest_set_json_packer) from one direct buffer of tableBytes bytes, little
 * endian as setStateWriter's table: i32 unknown_type, u32 discriminator length + its UTF-8 bytes, u32 n_events, then per event
 * u32 class-name length + its bytes, u32 event_type, u32 n_fields (at most 8), and per field u32 kind (SGR_JSON_*), u32 offset
 * (a record offset, or a program byte offset in state-topic mode), u32 PSTR slot bytes, u32 name length + its bytes. Every
 * string is copied out NUL-terminated; a name holding a NUL byte, a count out of range or a string past tableBytes throws
 * IllegalArgumentException. Returns the setter's code. */
#define JP_MAX_EVENTS 64
typedef int32_t (*packer_fn)(void* g, const char* disc, const sgr_json_event* events, uint32_t n_events, int32_t unknown_type);
typedef struct { const uint8_t* t; jlong n, at; char* arena; size_t used; const char* err; } TableReader;
static uint32_t tr_u32(TableReader* r) {
  uint32_t v = 0;
  if (r->err) return 0;
  if (r->n - r->at < 4) { r->err = "table: a field runs past tableBytes"; return 0; }
  memcpy(&v, r->t + r->at, 4);
  r->at += 4;
  return v;
}
static const char* tr_str(TableReader* r) {
  const uint32_t len = tr_u32(r);
  if (r->err) return "";
  if ((jlong)len > r->n - r->at) { r->err = "table: a string runs past tableBytes"; return ""; }
  char* s = r->arena + r->used;
  memcpy(s, r->t + r->at, len);
  s[len] = 0;
  if (strlen(s) != len) r->err = "table: a string holds a NUL byte";
  r->used += len + 1; r->at += len;
  return s;
}
static int32_t set_json_packer(JNIEnv* env, void* g, packer_fn set, jobject table, jlong table_bytes) {
  int ok = 1;
  if (table_bytes < 12) return bad_arg(env, "table: shorter than its header");
  const uint8_t* t = (const uint8_t*)direct(env, table, table_bytes, "table: direct buffer shorter than tableBytes", &ok);
  if (!ok) return SGR_ERR_INVALID;
  /* the strings, NUL-terminated: at most table_bytes bytes of text and one NUL per string (each string has a 4-byte length) */
  TableReader r = {t, table_bytes, 0, (char*)malloc((size_t)table_bytes + (size_t)table_bytes / 4 + 1), 0, 0};
  sgr_json_event* ev = (sgr_json_event*)calloc(JP_MAX_EVENTS, sizeof(sgr_json_event));
  if (!r.arena || !ev) { free(r.arena); free(ev); return bad_arg(env, "table: out of memory"); }
  const int32_t unknown_type = (int32_t)tr_u32(&r);
  const char* disc = tr_str(&r);
  const uint32_t n_events = tr_u32(&r);
  if (!r.err && n_events > JP_MAX_EVENTS) r.err = "table: more than 64 classes";
  for (uint32_t i = 0; !r.err && i < n_events; ++i) {
    ev[i].type_name = tr_str(&r);
    ev[i].event_type = tr_u32(&r);
    ev[i].n_fields = tr_u32(&r);
    if (!r.err && ev[i].n_fields > SGR_JSON_MAX_FIELDS) r.err = "table: more than 8 members in a class";
    for (uint32_t f = 0; !r.err && f < ev[i].n_fields; ++f) {
      const uint32_t kind = tr_u32(&r), off = tr_u32(&r);
      ev[i].fields[f].len = tr_u32(&r);
      ev[i].fields[f].name = tr_str(&r);
      if (!r.err && (kind > 255 || off > 0xffff)) r.err = "table: member kind or offset out of range";
      ev[i].fields[f].kind = (uint8_t)kind;
      ev[i].fields[f].dst_off = (uint16_t)off;
    }
  }
  const int32_t rc = r.err ? bad_arg(env, r.err) : set(g, disc, ev, n_events, unknown_type);
  free(r.arena);
  free(ev);
  return rc;
}
static int32_t ingest_packer(void* g, const char* d, const sgr_json_event* e, uint32_t n, int32_t u) { return sgr_ingest_set_json_packer((sgr_ingest*)g, d, e, n, u); }
static int32_t dingest_packer(void* g, const char* d, const sgr_json_event* e, uint32_t n, int32_t u) { return sgr_dingest_set_json_packer((sgr_dingest*)g, d, e, n, u); }
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_ingestSetJsonPacker(JNIEnv* env, jobject o, jlong g, jobject table, jlong table_bytes) {
  return set_json_packer(env, G(g), ingest_packer, table, table_bytes);
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_ingestSetAborted(JNIEnv* env, jobject o, jlong g, jint partition, jlongArray pids, jlongArray firsts) {
  jsize n = (*env)->GetArrayLength(env, pids);
  if ((*env)->GetArrayLength(env, firsts) != n) return bad_arg(env, "producerIds and firstOffsets differ in length");
  jlong* p = (*env)->GetLongArrayElements(env, pids, 0);
  jlong* f = (*env)->GetLongArrayElements(env, firsts, 0);
  int32_t rc = sgr_ingest_set_aborted(G(g), partition, (const int64_t*)p, (const int64_t*)f, (uint64_t)n);
  (*env)->ReleaseLongArrayElements(env, pids, p, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, firsts, f, JNI_ABORT);
  return rc;
}
JNIEXPORT jlong JNICALL Java_surge_gpu_Native_00024_ingestRecordBatches(JNIEnv* env, jobject o, jlong g, jint partition, jobject data, jlong nbytes) {
  sgr_ingest_stats st;
  int ok = 1; void* d = direct(env, data, nbytes, "data: direct buffer shorter than nbytes", &ok);
  if (!ok) return -1;
  int32_t rc = sgr_ingest_record_batches(G(g), partition, d, (uint64_t)nbytes, &st);
  if (rc != SGR_OK) {   /* a corrupt batch kills the stream thread, as a CorruptRecordException would */
    (*env)->ThrowNew(env, (*env)->FindClass(env, "java/lang/RuntimeException"), sgr_ingest_last_error(G(g)));
    return -1;
  }
  return (jlong)st.n_records;
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_foldIngested(JNIEnv* env, jobject o, jlong h, jlong g) { return sgr_fold_ingested(H(h), G(g)); }
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_growStates(JNIEnv* env, jobject o, jlong h, jlong n_agg) { return sgr_grow_states(H(h), (uint64_t)n_agg); }
JNIEXPORT jlongArray JNICALL Java_surge_gpu_Native_00024_ingestOffsets(JNIEnv* env, jobject o, jlong g, jint partition) {
  int64_t v[2] = {0, 0};
  sgr_ingest_offsets(G(g), partition, &v[0], &v[1]);
  jlongArray r = (*env)->NewLongArray(env, 2);
  (*env)->SetLongArrayRegion(env, r, 0, 2, (const jlong*)v);
  return r;
}

/* ---- device ingest: the same bytes, decoded on the GPU (include/sgr.h "device ingest") */
#define DG(g) ((sgr_dingest*)(intptr_t)(g))
JNIEXPORT jlong JNICALL Java_surge_gpu_Native_00024_dingestCreate(JNIEnv* env, jobject o, jlong h, jlong max_keys, jlong max_id_bytes) {
  sgr_dingest* g = 0;
  if (max_keys <= 0 || max_id_bytes < 0) { bad_arg(env, "maxKeys must be positive, maxIdBytes non-negative"); return 0; }
  int32_t rc = sgr_dingest_create(H(h), (uint64_t)max_keys, (uint64_t)max_id_bytes, &g);
  if (rc != SGR_OK) { (*env)->ThrowNew(env, (*env)->FindClass(env, "java/lang/RuntimeException"), "sgr_dingest_create failed (no device memory, or no engine)"); return 0; }
  return (jlong)(intptr_t)g;
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_dingestDestroy(JNIEnv* env, jobject o, jlong g) { return sgr_dingest_destroy(DG(g)); }
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_dingestSetNullValueType(JNIEnv* env, jobject o, jlong g, jint event_type) { return sgr_dingest_set_null_value_type(DG(g), event_type); }
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_dingestSetValueFraming(JNIEnv* env, jobject o, jlong g, jint framing) { return sgr_dingest_set_value_framing(DG(g), framing); }
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_dingestSetJsonPacker(JNIEnv* env, jobject o, jlong g, jobject table, jlong table_bytes) {
  return set_json_packer(env, DG(g), dingest_packer, table, table_bytes);
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_dingestSetStateTopic(JNIEnv* env, jobject o, jlong g, jint on) { return sgr_dingest_set_state_topic(DG(g), on); }
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_dingestSetAborted(JNIEnv* env, jobject o, jlong g, jint partition, jlongArray pids, jlongArray firsts) {
  jsize n = (*env)->GetArrayLength(env, pids);
  if ((*env)->GetArrayLength(env, firsts) != n) return bad_arg(env, "producerIds and firstOffsets differ in length");
  jlong* p = (*env)->GetLongArrayElements(env, pids, 0);
  jlong* f = (*env)->GetLongArrayElements(env, firsts, 0);
  int32_t rc = sgr_dingest_set_aborted(DG(g), partition, (const int64_t*)p, (const int64_t*)f, (uint64_t)n);
  (*env)->ReleaseLongArrayElements(env, pids, p, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, firsts, f, JNI_ABORT);
  return rc;
}
/* `data` must be a DIRECT buffer that stays untouched until dingestFold returns: the copy to the device is asynchronous.
 * Returns the number of data batches queued; throws on a malformed fetch (nothing of it is queued). */
JNIEXPORT jlong JNICALL Java_surge_gpu_Native_00024_dingestSubmit(JNIEnv* env, jobject o, jlong g, jint partition, jobject data, jlong nbytes) {
  sgr_ingest_stats st;
  int ok = 1; void* d = direct(env, data, nbytes, "data: direct buffer shorter than nbytes", &ok);
  if (!ok) return -1;
  int32_t rc = sgr_dingest_submit(DG(g), partition, d, (uint64_t)nbytes, &st);
  if (rc != SGR_OK) {
    (*env)->ThrowNew(env, (*env)->FindClass(env, "java/lang/RuntimeException"), sgr_dingest_last_error(DG(g)));
    return -1;
  }
  return (jlong)st.n_batches;
}
/* decode + intern + fold of everything submitted; Array(records folded, new aggregate ids). A corrupt batch fails the whole poll
 * (nothing applied, positions unchanged) and kills the consuming thread, as a CorruptRecordException would. */
JNIEXPORT jlongArray JNICALL Java_surge_gpu_Native_00024_dingestFold(JNIEnv* env, jobject o, jlong g) {
  sgr_ingest_stats st;
  int32_t rc = sgr_dingest_fold(DG(g), &st);
  if (rc != SGR_OK) {
    (*env)->ThrowNew(env, (*env)->FindClass(env, "java/lang/RuntimeException"), sgr_dingest_last_error(DG(g)));
    return 0;
  }
  int64_t v[2] = {(int64_t)st.n_records, (int64_t)st.n_new_keys};
  jlongArray r = (*env)->NewLongArray(env, 2);
  (*env)->SetLongArrayRegion(env, r, 0, 2, (const jlong*)v);
  return r;
}
JNIEXPORT jlongArray JNICALL Java_surge_gpu_Native_00024_dingestOffsets(JNIEnv* env, jobject o, jlong g, jint partition) {
  int64_t v[2] = {0, 0};
  sgr_dingest_offsets(DG(g), partition, &v[0], &v[1]);
  jlongArray r = (*env)->NewLongArray(env, 2);
  (*env)->SetLongArrayRegion(env, r, 0, 2, (const jlong*)v);
  return r;
}
JNIEXPORT jint JNICALL Java_surge_gpu_Native_00024_dingestReset(JNIEnv* env, jobject o, jlong g) { return sgr_dingest_reset(DG(g)); }
#endif
#endif
