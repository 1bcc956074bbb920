// zk_check.cuh — the self-check of the batched prover (include/zkattest.h, "Self-checked proving"): every proof a prove
// call wrote is verified with samples = sec_level before it leaves the library, and a proof that fails is released as
// FinalizeTask releases a row the prover itself rejected.
//
// The check's randomness is the seeded verifier rule (zk_seed.cuh) on c_b = SHA-256("ZKAttest/check/v1" || k_b), k_b being
// the 32-byte seed SeedProveTapeTask expanded for row b (the caller's or the hedged seed), or the first 96 bytes of the
// row's tape for a tape call (the blinders of comS1, keyXcom and keyYcom).
#pragma once
#include "zk_prove.cuh"
#include "zk_seed.cuh"
#include "zk_verify_agg.cuh"

namespace zk {

// One thread per row: c_b into seeds[b] (16-byte aligned rows of 32 bytes), and todo[b] = 1 when the prover gave the row
// status ZKA_OK (only those rows are checked; the others keep the prover's status)
struct CheckSeedTask {
  const uint8_t* key;     // k_b at key + b * key_stride
  size_t key_stride;
  int key_len;            // 32 (a seed) or 96 (three tape draws)
  const int32_t* status;  // [B] the prover's statuses, after FinalizeTask
  uint8_t* seeds;         // [B][32]
  uint8_t* todo;          // [B]
  ZK_HD void operator()(int b) const {
    Sha256 h;
    h.init();
    sha_tag(h, "ZKAttest/check/v1");
    h.update(key + (size_t)b * key_stride, key_len);
    sha_store(h, seeds + (size_t)32 * b);
    todo[b] = status[b] == ZKA_OK ? 1 : 0;
  }
};

// After the verifier's chain over the chunk: a checked row passes when the verifier gave ok = 1 and status ZKA_OK; any other
// verdict zeroes the row, sets its length to 0 and its status to ZKA_ERR_SELF_CHECK.  FIN_PARTS threads per row (as
// FinalizeTask); part 0 counts the row into counts[0] (checked) and counts[1] (failed).  The decision reads only todo / ok
// / vstatus, which no thread of this task writes.
struct CheckReleaseTask {
  const uint8_t* todo;       // [B] from CheckSeedTask
  const uint8_t* ok;         // [B] the verifier's verdicts
  const int32_t* vstatus;    // [B] the verifier's statuses
  uint8_t* proofs;           // [B][proof_stride]
  size_t proof_stride;
  uint32_t* proof_len;       // [B]
  int32_t* status;           // [B]
  uint32_t* counts;          // [2]
  ZK_HD void operator()(int t) const {
    const int b = t / FIN_PARTS, part = t % FIN_PARTS;
    if (!todo[b]) return;
    const bool pass = ok[b] == 1 && vstatus[b] == ZKA_OK;
    if (part == 0) {
      zk_atomic_add(counts, 1u);
      if (!pass) {
        zk_atomic_add(counts + 1, 1u);
        status[b] = ZKA_ERR_SELF_CHECK;
        proof_len[b] = 0;
      }
    }
    if (pass) return;
    uint8_t* row = proofs + (size_t)b * proof_stride;
    const size_t per = (proof_stride + FIN_PARTS - 1) / FIN_PARTS;
    size_t lo = per * part, hi = lo + per;
    if (hi > proof_stride) hi = proof_stride;
    for (size_t i = lo; i < hi; i++) row[i] = 0;
  }
};

}  // namespace zk
