// Host-side pieces of the block-level pre-pass (SURVEY.md section 8f rank 1, section 8a rows a11-a14).  The walk, the gates and the
// decisions run on the device (blockdev.cuh); what stays on the host is bookkeeping:
//   * split_block: find the envelopes of a serialized common.Block (the length-prefixed repeated field is inherently serial);
//   * MspTable / PolicyNode: the host copy of what fabgpu_msp_configure was given (re-issued to the device when key tables move);
//   * the validation codes the duplicate-tx-id pass needs (markTXIdDuplicates, core/committer/txvalidator/v20/validator.go:283-297).
// A host-thread implementation of the whole walk existed in round 1 as a cross-check (FABGPU_BLOCK_HOST=1); it was removed: the
// device logic itself is compiled for the host by the tests (tests/host_sim/blockdev_host.cpp) and checked there against the CPU restatement of the reference,
// and the library has no CPU path that could be mistaken for a fallback.  Host code only (no CUDA in this file).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace fabgpu { namespace blockval {

// peer.TxValidationCode (the ones the host pass touches)
enum : uint8_t { TX_VALID = 0, TX_DUPLICATE_TXID = 9, TX_NOT_VALIDATED = 254 };

struct Seg { uint32_t off = 0, len = 0; };                 // a byte range of the block buffer

// What the MSP serves in steady state (msp/cache), as handed to fabgpu_msp_configure.
struct MspTable {
    std::vector<std::string> serialized;                    // identity i's wire bytes
    std::vector<std::string> mspid;
    std::vector<uint8_t> keys_xy;                           // 64 bytes per identity
    std::vector<uint8_t> valid;                             // identity.Validate() outcome
    void add(const uint8_t* p, size_t n) { serialized.emplace_back((const char*)p, n); }
};

struct PolicyNode { int32_t type, n, first_child, n_children; };   // type 0: NOutOf(n) over children; 1: SignedBy(principal n); 2: ImplicitMeta(threshold n)

// Block{header = 1, data = 2, metadata = 3}, BlockData{repeated bytes data = 1} -> the envelopes' byte ranges.  false when the outer
// messages do not parse (Go: proto.Unmarshal of the Block fails).
bool split_block(const uint8_t* block, size_t len, std::vector<Seg>& envs);

} }  // namespace fabgpu::blockval
