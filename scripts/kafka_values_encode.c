/* kafka_values_encode.c — TEST INFRASTRUCTURE: producer-side RecordBatch v2 bytes of arbitrary key/value records, for
 * scripts/dingest_framing_bench.py (protobuf-wrapped and play-json event values at the e2e scale, where the pure-Python
 * encoder of oracle/kafka_batch.py would take hours).
 *
 * The batch layout, lz4 frame, CRC-32C and varints are oracle/kafka_encode.c's, included as they are, so both encoders write
 * the same framing; only the record key and value differ (given here instead of formatted from a Counter event). The script
 * compiles this file into a temporary directory at run time. */
#include "../oracle/kafka_encode.c"

/* Records i = 0..n-1 with key keys[key_offs[i], key_offs[i + 1]) and value vals[val_offs[i], val_offs[i + 1]) of ONE
 * partition, as consecutive RecordBatches of recs_per_batch records from base_offset. Returns the bytes written, -1 when `cap`
 * is too small, -2 when memory runs out. A bound for cap: the key and value bytes + 32 per record + 160 per batch, plus 1/255. */
/* nulls (optional): nulls[i] != 0 writes a null value for record i (a tombstone on a compacted topic; its value bytes are not read). */
int64_t kv_kafka_encode_values_nulls(const uint8_t* keys, const uint64_t* key_offs, const uint8_t* vals, const uint64_t* val_offs,
                                     const uint8_t* nulls, uint64_t n, uint32_t recs_per_batch, int lz4, int64_t base_offset, uint8_t* out,
                                     uint64_t cap) {
  if (!recs_per_batch) return -1;
  uint64_t body_cap = 0;
  uint8_t *body = NULL, *comp = NULL;
  uint64_t op = 0;
  const int64_t ts0 = 1600000000000ll;
  for (uint64_t s = 0; s < n; s += recs_per_batch) {
    const uint32_t cnt = (uint32_t)(n - s < recs_per_batch ? n - s : recs_per_batch);
    const uint64_t need = (key_offs[s + cnt] - key_offs[s]) + (val_offs[s + cnt] - val_offs[s]) + 32ull * cnt;
    if (need > body_cap) {
      free(body); free(comp);
      body_cap = need;
      body = (uint8_t*)malloc(body_cap);
      comp = (uint8_t*)malloc(body_cap + body_cap / 255 + 64 + 8 * (body_cap / 65536 + 1));
      if (!body || !comp) { free(body); free(comp); return -2; }
    }
    uint64_t bl = 0;
    for (uint32_t d = 0; d < cnt; d++) {
      const uint64_t i = s + d;
      const int null_value = nulls && nulls[i];
      const uint64_t kl = key_offs[i + 1] - key_offs[i], vl = null_value ? 0 : val_offs[i + 1] - val_offs[i];
      uint8_t head[24]; uint32_t h = 0;
      head[h++] = 0;                                   /* attributes */
      h += put_varlong(head + h, (int64_t)d);          /* timestampDelta */
      h += put_varint(head + h, (int32_t)d);           /* offsetDelta */
      uint8_t kv[10], vv[10];
      const uint32_t kh = put_varint(kv, (int32_t)kl), vh = put_varint(vv, null_value ? -1 : (int32_t)vl);
      const uint64_t r = h + kh + kl + vh + vl + 1;
      bl += put_varint(body + bl, (int32_t)r);
      memcpy(body + bl, head, h); bl += h;
      memcpy(body + bl, kv, kh); bl += kh; memcpy(body + bl, keys + key_offs[i], kl); bl += kl;
      memcpy(body + bl, vv, vh); bl += vh; memcpy(body + bl, vals + val_offs[i], vl); bl += vl;
      body[bl++] = 0;                                  /* headers */
    }
    const uint8_t* payload = body; uint64_t pl = bl;
    if (lz4) { pl = lz4_frame(body, bl, comp); payload = comp; }
    const uint64_t total = 61 + pl;
    if (op + total > cap) { free(body); free(comp); return -1; }
    uint8_t* b = out + op;
    be64(b, (uint64_t)(base_offset + (int64_t)s));
    be32(b + 8, (uint32_t)(total - 12));
    be32(b + 12, 0);                                   /* partitionLeaderEpoch */
    b[16] = 2;                                         /* magic */
    be16(b + 21, (uint16_t)(lz4 ? 3 : 0));             /* attributes */
    be32(b + 23, cnt - 1);                             /* lastOffsetDelta */
    be64(b + 27, (uint64_t)ts0); be64(b + 35, (uint64_t)(ts0 + cnt - 1));
    be64(b + 43, (uint64_t)-1ll); be16(b + 51, (uint16_t)-1); be32(b + 53, (uint32_t)-1);   /* producerId, epoch, baseSequence */
    be32(b + 57, cnt);
    memcpy(b + 61, payload, pl);
    be32(b + 17, crc32c(b + 21, total - 21));
    op += total;
  }
  free(body); free(comp);
  return (int64_t)op;
}

int64_t kv_kafka_encode_values(const uint8_t* keys, const uint64_t* key_offs, const uint8_t* vals, const uint64_t* val_offs, uint64_t n,
                               uint32_t recs_per_batch, int lz4, int64_t base_offset, uint8_t* out, uint64_t cap) {
  return kv_kafka_encode_values_nulls(keys, key_offs, vals, val_offs, NULL, n, recs_per_batch, lz4, base_offset, out, cap);
}
