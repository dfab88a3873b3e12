/*
 * program_oracle.c — compiled restatement of the fold-program semantics (include/sgr.h "fold program").
 * TEST INFRASTRUCTURE ONLY: never linked into or called from the product (surge_b200/).
 *
 * Line for line the same as oracle/program_interp.py (_handle, _equal, fold, fold_var, fold_arrival_order), so that the
 * CUDA kernels can be checked against the written semantics at sizes a Python loop cannot reach. Written from sgr.h and
 * the interpreter, never from the kernels. The rules around the fold are the reference's:
 *   events.foldLeft(state)(handleEvent)                      CommandModels.scala:25-28
 *   handler throws -> ACKError, the actor keeps its state    PersistentActor.scala:260-263,303-309
 *   publish iff newState != oldState (Double fields: ==)     PersistentActor.scala:252-257
 * Single-threaded: one pass over the log, a few nanoseconds per record.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { P_IF_EXISTS, P_MATERIALISE, P_CREATE, P_TOMBSTONE, P_THROW };
enum { P_OP_SET, P_OP_ADD_I32, P_OP_SUB_I32, P_OP_ADD_I64, P_OP_SUB_I64 };
enum { P_ST_EXISTS = 1, P_ST_CHANGED = 2, P_ST_ERROR = 4 };
#define P_MAX_TYPES 16
#define P_MAX_OPS 8
#define P_MAX_STATE 128

/* The program as a flat u32 array (oracle/program_interp.py packs it): one layout, no struct padding questions. */
typedef struct {
  uint32_t state_bytes, n_types, n_f64;
  uint32_t f64_off[8];
  uint32_t exists[P_MAX_TYPES];
  uint32_t n_ops[P_MAX_TYPES];
  uint32_t ops[P_MAX_TYPES][P_MAX_OPS][4];   /* opcode, dst, src, len */
} orc_program;

static uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
static void wr32(uint8_t* p, uint32_t v) { memcpy(p, &v, 4); }
static void wr64(uint8_t* p, uint64_t v) { memcpy(p, &v, 8); }

/* Option[State] with JVM object identity reduced to one bit: `fresh` is set once an applied event built a new instance
 * (a rule with field ops, CREATE, MATERIALISE on None). The actor's own instance is the prior state; `cur eq old` holds
 * exactly while no applied event built a new one (a TOMBSTONE makes cur None, and only a new instance makes it Some again). */
typedef struct {
  int has;
  int fresh;
  uint8_t b[P_MAX_STATE];
} opt_state;

/* _handle: 0 = applied, 1 = the handler threw. Checks in the interpreter's order: MatchError, THROW, TOMBSTONE, then the
 * short-record check (variable records), then the exists rule, then the ops. */
static int handle(const orc_program* p, uint32_t user, opt_state* s, const uint8_t* rec, uint64_t avail) {
  const uint32_t etype = rd32(rec);
  if (etype >= p->n_types) return 1;                 /* scala.MatchError */
  const uint32_t ex = p->exists[etype], nops = p->n_ops[etype];
  if (ex == P_THROW) return 1;
  if (ex == P_TOMBSTONE) { s->has = 0; memset(s->b, 0, user); return 0; }
  for (uint32_t i = 0; i < nops; i++)
    if ((uint64_t)p->ops[etype][i][2] + p->ops[etype][i][3] > avail) return 1;   /* record too short for this class */
  if (ex == P_IF_EXISTS) {
    if (!s->has) return 0;
    if (!nops) return 0;                              /* `current`: the same instance */
  } else if (ex == P_MATERIALISE) {
    if (s->has && !nops) return 0;
    if (!s->has) memset(s->b, 0, user);
  } else {                                            /* CREATE */
    memset(s->b, 0, user);
  }
  s->has = 1;
  s->fresh = 1;
  for (uint32_t i = 0; i < nops; i++) {
    const uint32_t opc = p->ops[etype][i][0], dst = p->ops[etype][i][1], src = p->ops[etype][i][2], ln = p->ops[etype][i][3];
    switch (opc) {
      case P_OP_SET: memmove(s->b + dst, rec + src, ln); break;
      case P_OP_ADD_I32: wr32(s->b + dst, rd32(s->b + dst) + rd32(rec + src)); break;
      case P_OP_SUB_I32: wr32(s->b + dst, rd32(s->b + dst) - rd32(rec + src)); break;
      case P_OP_ADD_I64: wr64(s->b + dst, rd64(s->b + dst) + rd64(rec + src)); break;
      default:           wr64(s->b + dst, rd64(s->b + dst) - rd64(rec + src)); break;
    }
  }
  return 0;
}

/* _equal: Option equality; case-class equals starts with `this eq that`; Double fields compare with JVM == (0.0 == -0.0,
 * NaN != NaN), every other byte bitwise. */
static int equal(const orc_program* p, uint32_t user, const opt_state* old, const opt_state* cur) {
  if (old->has != cur->has) return 0;
  if (!old->has || !cur->fresh) return 1;
  uint8_t skip[P_MAX_STATE];
  memset(skip, 0, sizeof skip);
  for (uint32_t f = 0; f < p->n_f64; f++) {
    const uint32_t off = p->f64_off[f];
    double x, y;
    memcpy(&x, old->b + off, 8); memcpy(&y, cur->b + off, 8);
    if (!(x == y)) return 0;
    memset(skip + off, 1, 8);
  }
  for (uint32_t i = 0; i < user; i++)
    if (!skip[i] && old->b[i] != cur->b[i]) return 0;
  return 1;
}

static void load_prior(uint32_t sb, const uint8_t* row, opt_state* s) {
  memset(s, 0, sizeof *s);
  if (row && (rd32(row + sb - 8) & P_ST_EXISTS)) { s->has = 1; memcpy(s->b, row, sb - 8); }
}

static void store(const orc_program* p, const opt_state* old, const opt_state* cur, int threw, uint64_t k, uint8_t* out) {
  const uint32_t sb = p->state_bytes, user = sb - 8;
  const opt_state* fin = threw ? old : cur;
  uint32_t flags = threw ? P_ST_ERROR : (equal(p, user, old, cur) ? 0u : P_ST_CHANGED);
  memset(out, 0, sb);
  if (fin->has) { memcpy(out, fin->b, user); flags |= P_ST_EXISTS; }
  wr32(out + user, flags);
  wr32(out + user + 4, threw ? (uint32_t)k : 0u);
}

static int check_program(const orc_program* p) {
  if (p->state_bytes < 16 || p->state_bytes > P_MAX_STATE || p->state_bytes % 16) return -1;
  if (p->n_types == 0 || p->n_types > P_MAX_TYPES || p->n_f64 > 8) return -1;
  const uint32_t user = p->state_bytes - 8;
  for (uint32_t f = 0; f < p->n_f64; f++) if (p->f64_off[f] + 8 > user) return -1;
  for (uint32_t t = 0; t < p->n_types; t++) {
    if (p->exists[t] > P_THROW || p->n_ops[t] > P_MAX_OPS) return -1;
    for (uint32_t i = 0; i < p->n_ops[t]; i++) {
      const uint32_t* o = p->ops[t][i];
      if (o[0] > P_OP_SUB_I64 || o[1] + o[3] > user) return -1;
      if ((o[0] == P_OP_ADD_I32 || o[0] == P_OP_SUB_I32) && o[3] != 4) return -1;
      if ((o[0] == P_OP_ADD_I64 || o[0] == P_OP_SUB_I64) && o[3] != 8) return -1;
    }
  }
  return 0;
}

/* fold: fixed 64-byte records in CSR order; seg_offsets are byte offsets (n_agg + 1), multiples of 16 apart, the first
 * one need not be 0. Each segment's whole records fold at their own byte positions; a trailing 16, 32 or 48 bytes is a
 * malformed event: the handler throws there, at err_idx = the number of whole records (include/sgr.h).
 * initial: prior table or NULL (None everywhere). n_events counts the events applied (those after a throw are dropped). */
int orc_prog_fold(const orc_program* p, const uint8_t* records, const uint64_t* seg_offsets, uint64_t n_agg,
                  const uint8_t* initial, uint8_t* out, uint64_t* n_events, uint64_t* n_errors) {
  if (check_program(p)) return -1;
  for (uint32_t t = 0; t < p->n_types; t++)
    for (uint32_t i = 0; i < p->n_ops[t]; i++) if (p->ops[t][i][2] + p->ops[t][i][3] > 64) return -1;
  const uint32_t sb = p->state_bytes;
  const uint64_t base = seg_offsets[0];   /* `records` starts at the first segment */
  uint64_t nev = 0, nerr = 0;
  for (uint64_t i = 0; i < n_agg; i++) {
    const uint64_t lo = seg_offsets[i], hi = seg_offsets[i + 1];
    if (hi < lo || (lo - base) % 16 || (hi - base) % 16) return -1;
    opt_state old, cur;
    load_prior(sb, initial ? initial + i * sb : NULL, &old);
    cur = old;
    int threw = 0;
    uint64_t k = 0;
    for (uint64_t pos = lo - base; pos < hi - base; pos += 64, k++)
      if (hi - base - pos < 64 || handle(p, sb - 8, &cur, records + pos, 64)) { threw = 1; break; }
    store(p, &old, &cur, threw, k, out + i * sb);
    nev += k; nerr += (uint64_t)threw;
  }
  if (n_events) *n_events = nev;
  if (n_errors) *n_errors = nerr;
  return 0;
}

/* fold_var: SGR_REC_VAR16 records {type, seq, payload_len, agg} + payload padded to 16 bytes. A record that does not fit
 * its segment, is longer than max_record_bytes (header included, before padding) or is too short for the ops of its
 * event class is a malformed event: the handler throws at that record. */
int orc_prog_fold_var(const orc_program* p, uint32_t max_record_bytes, const uint8_t* log, const uint64_t* seg_offsets,
                      uint64_t n_agg, const uint8_t* initial, uint8_t* out, uint64_t* n_events, uint64_t* n_errors) {
  if (check_program(p)) return -1;
  const uint32_t sb = p->state_bytes;
  uint64_t nev = 0, nerr = 0;
  for (uint64_t i = 0; i < n_agg; i++) {
    uint64_t pos = seg_offsets[i];
    const uint64_t end = seg_offsets[i + 1];
    if (end < pos) return -1;
    opt_state old, cur;
    load_prior(sb, initial ? initial + i * sb : NULL, &old);
    cur = old;
    int threw = 0;
    uint64_t k = 0;
    while (pos < end) {
      if (end - pos < 16) { threw = 1; break; }
      const uint64_t plen = rd32(log + pos + 8);
      const uint64_t rlen = 16 + ((plen + 15) / 16) * 16;
      if (16 + plen > max_record_bytes || rlen > end - pos) { threw = 1; break; }
      if (handle(p, sb - 8, &cur, log + pos, 16 + plen)) { threw = 1; break; }
      pos += rlen;
      k++;
    }
    store(p, &old, &cur, threw, k, out + i * sb);
    nev += k; nerr += (uint64_t)threw;
  }
  if (n_events) *n_events = nev;
  if (n_errors) *n_errors = nerr;
  return 0;
}

/* fold_arrival_order: one micro-batch in arrival order onto a live table (records carry the aggregate index at +8, u64).
 * Per-batch flags of every slot are cleared first; the records are grouped stably by aggregate and each touched
 * aggregate folds its records onto its row. table == the prior table on entry, the result on return. Returns -1 (and
 * leaves the table as it was) when a record names an aggregate >= n_agg. */
int orc_prog_fold_arrival(const orc_program* p, const uint8_t* records, uint64_t n, uint8_t* table, uint64_t n_agg,
                          uint64_t* n_events, uint64_t* n_errors) {
  if (check_program(p)) return -1;
  for (uint32_t t = 0; t < p->n_types; t++)
    for (uint32_t i = 0; i < p->n_ops[t]; i++) if (p->ops[t][i][2] + p->ops[t][i][3] > 64) return -1;
  const uint32_t sb = p->state_bytes, user = sb - 8;
  for (uint64_t r = 0; r < n; r++) if (rd64(records + r * 64 + 8) >= n_agg) return -1;
  uint64_t* first = (uint64_t*)calloc(n_agg + 1, sizeof(uint64_t));
  uint64_t* order = (uint64_t*)malloc((n ? n : 1) * sizeof(uint64_t));
  uint8_t* seg = (uint8_t*)malloc((n ? n : 1) * 64);
  if (!first || !order || !seg) { free(first); free(order); free(seg); return -2; }
  for (uint64_t r = 0; r < n; r++) first[rd64(records + r * 64 + 8) + 1]++;
  for (uint64_t a = 0; a < n_agg; a++) first[a + 1] += first[a];
  for (uint64_t r = 0; r < n; r++) order[first[rd64(records + r * 64 + 8)]++] = r;   /* stable: arrival order kept */
  for (uint64_t a = n_agg; a > 0; a--) first[a] = first[a - 1];
  first[0] = 0;
  for (uint64_t j = 0; j < n; j++) memcpy(seg + j * 64, records + order[j] * 64, 64);
  for (uint64_t a = 0; a < n_agg; a++) {
    uint8_t* row = table + a * sb;
    wr32(row + user, rd32(row + user) & P_ST_EXISTS);
    wr32(row + user + 4, 0);
  }
  uint64_t nev = 0, nerr = 0;
  uint8_t prior[P_MAX_STATE];
  for (uint64_t a = 0; a < n_agg; a++) {
    if (first[a + 1] == first[a]) continue;
    const uint64_t off[2] = {first[a] * 64, first[a + 1] * 64};
    uint64_t ne = 0, nr = 0;
    memcpy(prior, table + a * sb, sb);
    orc_prog_fold(p, seg + off[0], off, 1, prior, table + a * sb, &ne, &nr);
    nev += ne; nerr += nr;
  }
  free(first); free(order); free(seg);
  if (n_events) *n_events = nev;
  if (n_errors) *n_errors = nerr;
  return 0;
}
