// Arguments of the FT-ZeRO-1 replica audit kernels (audit.cu). parallel/zero1.py builds the digest table and decodes the
// report; the layouts here and there must stay in sync.
#pragma once
#include "common.cuh"

namespace tft {
namespace audit {

// One row of the digest kernel's table, eight 64-bit fields (Python builds them as an int64 tensor): the 8-byte words
// [word0, word0 + nwords) of one array, by GLOBAL word index (word i is bytes [8 i, 8 i + 8) of the flat vector's byte
// image), are digested with `seed` and added into slots[slot]. word0 is even (the range starts on a 16-byte vector).
// Flat arrays pass their base (global index 0) and no table; paged arrays pass the pool and the page table, and global
// byte g then lives at pool byte (table[g >> page_byte_shift] << page_byte_shift) | (g & (page bytes - 1)).
struct DigestEntry {
  const char* base;
  const int* table;         // nullptr: flat
  uint64_t page_byte_shift; // log2 of a page's bytes (paged only); a page is at least 16 bytes
  uint64_t word0;
  uint64_t nwords;
  uint64_t seed;
  uint64_t slot;
  uint64_t chunk0;          // index of this row's first chunk of kDigestChunkWords words
};

constexpr size_t kDigestChunkWords = 8192;  // 64 KiB per chunk: one table lookup and one warp atomic per chunk and warp

// The one-CTA comparison of a quorum's digests. Rank r's z1_audit segment holds, for unit u, its weights digest at slot
// u * stride and the digest of array a of its j-th held slice (slice rank - j) at u * stride + 1 + j * narrays + a, and
// its update count at slot nunits * stride.
struct CompareArgs {
  PeerTable pt;                 // data[] = every rank's z1_audit segment
  StatusBlock* st;
  const int* ok;                // result of the handshake in front of the kernel
  unsigned long long* report;   // host-mapped: kReportHeader words, then world x (nunits * stride + 1) slots
  uint64_t seq;                 // audit sequence number, written to the report last
  int nunits;
  int stride;                   // slots per unit
  int k;                        // holders per slice (1: weights only)
  int narrays;                  // state arrays digested per held slice (master, m, v and the EMA when kept)
};

// report[0] = seq, [1] = groups whose digests disagree, [2] = world, [3] = slots per rank
constexpr int kReportHeader = 4;

}  // namespace audit
}  // namespace tft
