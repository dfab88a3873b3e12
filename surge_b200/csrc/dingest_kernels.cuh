// dingest_kernels.cuh — device-side decode of Kafka record batches (launch interface of dingest_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "devbuf.h"
#include "id_dict.cuh"
#include "value_framing.h"

namespace sgr {

// error codes a kernel leaves in DgBatch::err or, for one record, in DgBatch::rec_err (0 = fine); dingest.cu turns them into messages
enum DgErr : uint32_t {
  DG_OK = 0, DG_CRC = 1, DG_LZ4_HEADER = 2, DG_LZ4_BLOCK = 3, DG_LZ4_SEQUENCE = 4, DG_LZ4_CHECKSUM = 5, DG_LZ4_TOO_LARGE = 6,
  DG_RECORD_LENGTH = 7, DG_RECORD_MALFORMED = 8, DG_RECORD_COUNT = 9, DG_VALUE_LENGTH = 10, DG_ID_LENGTH = 11, DG_STRAY_BYTES = 12,
  DG_ARENA_FULL = 13,   // not a data error: the batch's arena claim did not fit (the host lays the arena out exactly and repeats)
  DG_VALUE_FRAMING = 14,   // a protobuf / JSON value was refused: the code is DG_VALUE_FRAMING | vf::Reason << 8
  DG_STATE_LENGTH = 15,    // state topic: a value longer than the program bytes; the code is DG_STATE_LENGTH | min(length, 2^24 - 1) << 8
};

// One data batch that survived the host's header walk (control batches, aborted transactions and anything below the partition's
// position never reach the device).
struct DgBatch {
  uint64_t src_off;      // byte offset of the batch (its baseOffset field) inside the wire buffer
  int64_t base_offset;   // first offset of the batch
  int64_t min_offset;    // records below this offset were decoded by an earlier call: duplicates, dropped
  uint32_t total_len;    // 12 + batchLength
  uint32_t n_records;    // recordsCount of the header
  uint32_t stored_crc;   // CRC-32C field of the header
  uint32_t rec_base;     // index of the batch's first record in the per-record tables
  uint32_t dsize;        // out (size pass): decompressed bytes of the records section (lz4), else its stored length
  uint16_t codec;        // 0 none, 3 lz4
  uint16_t err;          // out: DgErr of the batch as a whole (CRC, lz4, the record walk); parse runs only when it is 0
  uint64_t arena_off;    // in (decode pass): where the decompressed section goes
  // out: (record << 32) | DgErr of the record an error refers to, ~0 for none (set by the walk). The walk's own errors name
  // their record here; a parse thread that refuses its record takes the atomicMin, so the batch reports its LOWEST refused
  // record, the one the host decoder, which checks records in order, stops at
  unsigned long long rec_err;
};
static_assert(sizeof(DgBatch) == 64, "one descriptor per 64 bytes: the descriptor arrays cross PCIe every poll");
constexpr unsigned long long kNoRecErr = ~0ull;

struct DgParse {
  const uint8_t* wire;
  const uint8_t* arena;
  DgBatch* batches;
  uint32_t n_batches;
  uint32_t rec_begin;            // first record slot this launch parses
  uint32_t n_records;            // one past the last record slot this launch parses
  const uint32_t* rec_off;       // [n_records] offset of the record (its length varint) inside the batch's records section
  const uint32_t* rec_batch;     // [n_records] batch of the record
  uint8_t* out;                  // [n_records] packed 64-byte records; dropped records become holes (agg == ~0)
  int32_t null_value_type;       // -1: keyed records with a null value are dropped; else they become events of this type
  DgDict dict;
  int32_t value_framing;         // SGR_VALUE_*: how a value wraps the packed event (selects the kernel's instantiation)
  vf::Table json;                // SGR_VALUE_JSON: the registered member table, in device memory
  // state topic (sgr_dingest_set_state_topic): `out` holds rows of row_bytes (state_bytes - 8) program bytes instead of packed
  // records, with each slot's dense index (~0u: a hole) in idx and 0 (tombstone) / 1 (row) in present
  bool state_topic;
  uint32_t row_bytes;
  uint32_t* idx;
  uint8_t* present;
};

cudaError_t dg_launch_parse(const DgParse& p, cudaStream_t st);
// nbytes rounded up to 16: both buffers need that much room; host_mapped is the DEVICE address of page-locked, mapped host memory
cudaError_t dg_copy_from_mapped_host(const void* host_mapped, void* dst, uint64_t nbytes, cudaStream_t st);
cudaError_t dg_prepare();   // uploads the CRC tables (a synchronous copy: call it before anything runs on other streams)
// The two thread-per-batch kernels read wire and arena through a ring that runs up to 256 bytes past a batch's last byte: both
// buffers need that much room past their content.
// With arena_ctl, every lz4 batch claims claim_mult x its compressed size of arena.
cudaError_t dg_launch_crc_size_fast(const uint8_t* wire, DgBatch* batches, uint32_t n, unsigned long long* arena_ctl, uint32_t claim_mult, cudaStream_t st);
// batches: the sub-array to process (n of them), whose first element has index `index_base` in the full array (what rec_batch records);
// arena_ctl as given to dg_launch_crc_size_fast for the same batches (nullptr: dsize is exact, not a slot capacity)
cudaError_t dg_launch_decode_walk_fast(const uint8_t* wire, uint8_t* arena, DgBatch* batches, uint32_t n, uint32_t index_base, uint32_t* rec_off, uint32_t* rec_batch,
                                       unsigned long long* arena_ctl, cudaStream_t st);
cudaError_t dg_gather_keys(const DgDict& d, uint64_t from, uint32_t n, uint32_t* d_offs, uint8_t* d_bytes, DevBuf& scan_tmp, cudaStream_t st);

}  // namespace sgr
