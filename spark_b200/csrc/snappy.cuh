// snappy.cuh -- Snappy page bodies of a Parquet column chunk -> a device image of the decoded pages (snappy.cu), and the
// per-page records the host reads back to describe the image (sb_scan_decode_compressed in scan.cu).
#pragma once
#include "common.cuh"

namespace sb {

// one page of a call: [levels_bytes uncompressed level bytes (V2)][values: a raw Snappy block, or stored as they are]
struct SnappyPage {
  const uint8_t *src;        // device: the page body as it lies in the chunk
  uint8_t *dst;              // device: the page's place in the image (dst_bytes long)
  int64_t levels_bytes;      // copied as they are in front of the values
  int64_t src_bytes, dst_bytes;
  int32_t compressed;        // 0: the values are stored as they are (src_bytes == dst_bytes)
  int32_t slot;              // index of the page's status / record
};

// what the host needs of one decoded page to build its sb_page: the Snappy status, a V1 page's definition-level length and the
// first bytes of the values section (a DELTA_* header is at most four 10-byte varints)
constexpr int PAGE_HEAD_BYTES = 48;
struct PageRecord {
  int32_t status;            // SNAPPY_* below
  uint32_t def_len;          // V1 page with definition levels: the 4-byte length in front of them
  int32_t body_short;        // V1 page with definition levels shorter than that 4-byte length
  int32_t head_bytes;        // valid bytes of head
  uint8_t head[PAGE_HEAD_BYTES];
};
struct ResolveTask {
  const uint8_t *image;      // device: the decoded page
  int64_t bytes;             // its decoded size
  int64_t levels_bytes;      // V2: level bytes in front of the values
  int32_t v1_def;            // V1 page of an optional column: the body starts with [4-byte length][levels]
  int32_t slot;
};

enum SnappyStatus {
  SNAPPY_OK = 0,
  SNAPPY_BAD_PREAMBLE = 1,     // truncated or overlong length preamble
  SNAPPY_LENGTH_MISMATCH = 2,  // preamble != the page header's uncompressed size
  SNAPPY_INPUT_OVERRUN = 3,    // a tag, its extra bytes or a literal past the end of the input
  SNAPPY_BAD_OFFSET = 4,       // copy offset 0 or reaching before the page's first byte
  SNAPPY_OUTPUT_OVERRUN = 5,   // an element writes past the declared length
  SNAPPY_LEFTOVER = 6,         // input left over once the declared length is produced
  SNAPPY_SHORT = 7,            // input ends before the declared length is produced
};
const char *snappy_status_text(int status);

// scan_snappy (one block per page, in the order given: the host sorts them largest first) and scan_resolve_pages (one thread per
// page); both asynchronous on st
void launch_snappy(const SnappyPage *d_pages, int npages, int32_t *d_status, cudaStream_t st);
void launch_resolve_pages(const ResolveTask *d_tasks, int ntasks, const int32_t *d_status, PageRecord *d_records, cudaStream_t st);

}  // namespace sb
