/* zkattest.h — C ABI of libzkattest, the H100-native ZKAttest prover/verifier.
 *
 * Drop-in boundary for the hot path of cloudflare/zkp-ecdsa v0.2.6.  The reference has no
 * FFI of its own (pure TypeScript); these entry points are what a node-addon-api shim
 * binds so that the three public functions keep their TypeScript signatures
 * (INTEGRATION.md shows the shim):
 *
 *   zka_params_generate  <-> generateParamsList   /root/reference/src/zkpAttestList.ts:88-92
 *   zka_prove_batch      <-> proveSignatureList   /root/reference/src/zkpAttestList.ts:104-145
 *   zka_verify_batch     <-> verifySignatureList  /root/reference/src/zkpAttestList.ts:147-184
 *   zka_key_to_int       <-> keyToInt             /root/reference/src/zkpAttestList.ts:94-102
 *
 * All integers and points cross the boundary in the reference's own encodings:
 *   Group.Point.toBytes():  P-256 0x04||x||y = 65 B (weier.ts:244-255),
 *                           tomEdwards256 0x04||x||y = 67 B (edwards.ts:195-203)
 *   Group.Scalar.toBytes(): big-endian, 32 B (p256) / 33 B (tomEdwards256) (group.ts:196-199)
 *   bigint ring entries:    32-byte big-endian (keyToInt output, < 2^256)
 *
 * Flat proof layout (the reference only has typedjson JSON, serde.ts:21-36; field order is
 * that of the reference classes):
 *   proof   := R(65) comS1(65) keyXcom(67) keyYcom(67) rep[SecLevel] GK     zkpAttestList.ts:30-35
 *   rep     := tag(1) A(65) Tx(67) Ty(67) body                              exp.ts:27-40
 *   body    := tag==1: alpha(32) beta1(32) beta2(33) beta3(33)
 *              tag==0: z(32) z2(32) PointAddProof(3266) r1(33) r2(33)
 *   PointAddProof := C_8 C_10 C_11 C_13 pi_8 pi_10 pi_11 pi_13 pi_x pi_y     pointAdd.ts:29-38
 *   MultProof(633)     := C_4 A_x A_y A_z A_4_1 A_4_2 t_x t_y t_z t_rx t_ry t_rz t_r4   mult.ts:27-39
 *   EqualityProof(233) := A_1 A_2 t_x t_r1 t_r2                              equality.ts:28-32
 *   GK      := n(1) cl[n] ca[n] cb[n] cd[n] f[n] za[n] zb[n] zd              gk.ts:32-39
 *
 * Randomness.  The reference draws from crypto.getRandomValues inside rnd() (big.ts:171-181).
 * Here the caller supplies the randomness as a TAPE of 32-byte big-endian draws per proof, in
 * the reference's call order (SURVEY.md 3.1):
 *   prove:  [0] comS1.r (mod p256.n)  [1],[2] keyXcom.r, keyYcom.r (mod tom.order)
 *           [3+4i..6+4i] alpha_i, r_i (mod p256.n), Tx_i.r, Ty_i.r (mod tom.order), i < SecLevel
 *           then 40 draws (mod tom.order) per 0-bit repetition in index order, then 5 per GK round.
 *           Total 3 + 4*SecLevel + 40*Z + 5*n draws; zka_prove_tape_len() gives the worst case.
 *   Every draw must already be below its modulus (rnd()'s rejection loop is done by the host:
 *   the modulus of draw k depends only on k); otherwise status = ZKA_ERR_TAPE_RANGE.
 *
 * Seeded randomness (zka_prove_batch_seeded, zka_verify_batch_seeded, zka_seed_tape).  Instead of a tape the caller
 * gives 32 seed bytes per proof and the library expands the tape on the GPU.  The expansion is a ChaCha20 keystream
 * (RFC 8439 2.3: 20 rounds, little-endian words, 32-bit block counter from 0) keyed by the seed, with the 96-bit nonce
 * le32(domain) || le64(index); stream(seed, domain, index) = its blocks 0, 1, 2, ... concatenated.
 *   prover draw k (tape order above, k < 3 + 44S + 5n): rnd(modulus of draw k) on stream(seed, 1, k) — 32 bytes at a
 *     time read as a big-endian integer, the first one below the modulus kept — gives tape bytes [32k, 32k + 32).
 *   verifier 32-byte slot t (the 2n + 1 GK drains, then the 25 * samples packed exp drains, in layout order): the first
 *     32-byte candidate of stream(seed, 2, t) below p256.n.  p256.n is the smaller modulus; one bound serves every slot,
 *     as the modulus of a packed drain depends on challenge bits (a 2^-32 relaxation of rnd() that does not affect the
 *     soundness of the random linear combination).
 *   verifier index byte i (i < S - 2): rnd(S - i) on stream(seed, 3, i), one byte per candidate; the pad bytes are zero.
 * A seeded call is byte-identical to the tape call on zka_seed_tape's expansion of the same seeds.
 * A SEED IS AS SECRET AS THE WITNESS AND MUST BE FRESH FOR EVERY PROOF: two proofs of different statements made from one
 * seed share every alpha_i; a repetition that reveals alpha_i in one and z = alpha_i - s1 in the other gives s1, and then
 * pk = s1 * R - Q: the signer is deanonymised.  The domains keep a seed's prover and verifier streams apart; they do not
 * make reuse safe.  Draw seeds from the OS CSPRNG.
 *
 * Hedged seeds (zka_prove_batch_hedged, zka_prove_batch_rings_hedged, zka_hedge_seeds[_rings]).  The seed of each row is
 * derived on the GPU from the caller's seed, the statement and the signature (as RFC 6979 and its hedged variants derive
 * a signature nonce), and then expanded by the seeded rule above.  Byte strings, || = concatenation:
 *   params digest  SHA-256("ZKAttest/hedge/params/v1" || proof-group name, NUL-padded to 16 bytes || h_nist (65) ||
 *                  h_proof (point_bytes) || le32(sec_level)), computed once by zka_params_create.
 *   ring digest    of a ring of N entries, depth n = ceil(log2 N): e_j = ring[j] mod the proof-group order as 32 bytes
 *                  big-endian for j < 2^n, the padding entries being e_0 (gk.ts:75-86); leaf k = SHA-256(e_{1024k} || ... ||
 *                  e_{1024k+1023}), one leaf of all 2^n entries when 2^n <= 1024; digest = SHA-256("ZKAttest/hedge/ring/v1" ||
 *                  le32(N) || le32(n) || leaf_0 || leaf_1 || ...).  Computed on the GPU once per one-ring call, and for every
 *                  ring of a set once by zka_rings_create.
 *   row seed       SHA-256("ZKAttest/hedge/prove/v1" || params digest || ring digest of the row's ring || seed_b (32, or 32
 *                  zero bytes when seeds == NULL) || msg_hash_b (32) || sig_b (64) || pk_b (65) || le32(which_b)).
 * Neither the row's index in the call nor its neighbours are hashed: rows in any order give the same bytes.  A hedged call
 * is byte-identical (proofs, proof_len, status and its precedence) to the seeded call on the seeds zka_hedge_seeds returns.
 * Two rows share randomness only if every hashed input is equal; they then prove the same statement with the same witness,
 * and their proof bytes are identical.  So a caller seed that repeats (a broken CSPRNG, a VM restored from a snapshot, a
 * forked worker, a reused buffer) no longer deanonymises the signer.  With seeds == NULL the proofs are deterministic and
 * their randomness rests on the secrecy of the signature alone: (r, s) with the message recovers the public key, so the
 * signature is as secret as the witness.  Derived seeds stay in library workspace; only zka_hedge_seeds copies them out.
 *
 * Self-checked proving (zka_set_option(ctx, "self_check", 2); 1 = off, the default).  A fault during a prove call (one
 * wrong commitment byte) changes the challenge of that run; a deterministic prover that also makes the correct proof of
 * the same statement then reveals alpha_i in one and z = alpha_i - s1 in the other, as a reused seed does.  With the check
 * on, every row of the six batched proveSignatureList calls (zka_prove_batch[_seeded|_hedged], zka_prove_batch_rings[_seeded|
 * _hedged]) whose prover status is ZKA_OK is verified before the call releases it: verifySignatureList on the row's own
 * ring with samples = sec_level, i.e. EVERY repetition (a faulty repetition missed by a partial check is exactly the one
 * that leaks).  It also catches a `which` that is inside the ring but not the signer's key, which the reference proves
 * without complaint.  A row passes when the check gives ok = 1 and status 0: its proof bytes, proof_len and status are
 * those of the unchecked call.  Any other verdict (a verifier status included) gives the row ZKA_ERR_SELF_CHECK, its
 * bytes zeroed and proof_len 0, as for a row the prover rejected.  The check's randomness, so that a checked call can be
 * reproduced:
 *   k_b  the 32-byte seed expanded for row b (seeded calls: the caller's seed; hedged calls: the derived seed), or for a
 *        tape call the row's first 96 tape bytes (the blinders of comS1, keyXcom and keyYcom)
 *   c_b  SHA-256("ZKAttest/check/v1" || k_b)
 * and the verdict of row b is that of zka_verify_batch_seeded (zka_verify_batch_rings_seeded for a set) with
 * samples = sec_level and seeds c on the unchecked proofs.  c_b IS AS SECRET AS THE WITNESS, like the seed it comes from;
 * it stays in library workspace.  Checked calls are deterministic wherever the unchecked call is.  The check runs per
 * chunk on the device, behind the prover's last kernel: no proof byte crosses PCIe twice, and a chunk reported by
 * zka_set_progress holds checked proofs only.  zka_stat counts "self_check_rows" and "self_check_fail".  The stand-alone
 * sub-proof provers (zka_prove_exp_batch, zka_prove_membership_batch, zka_prove_equality_batch, zka_prove_mult_batch,
 * zka_prove_pointadd_batch) are never checked.
 *
 * Traceable proofs (zka_prove_batch_traced[_seeded], zka_verify_batch_traced[_seeded], zka_open_batch).  An opener with
 * the key sk in [1, q) and Y = sk g (zka_trace_pubkey) can say which ring member made a traced proof; without sk the proof
 * stays anonymous in its ring.  g, h are the proof group's generator and params' ProofGroup.h, q its order (= p256.p), PB /
 * SB its point / scalar bytes (67 / 33 tomEdwards256, 65 / 32 war256), || concatenation.  A traced row is the untraced row
 * of the same call, byte for byte, followed by a trace block of zka_trace_len() = 5 PB + 3 SB bytes (434 / 421):
 *   witness   x = the x-coordinate of pk (the value keyXcom commits to), r = the blinder of keyXcom (prover draw 1)
 *   draws     k, a, beta, c in [0, q): tape calls read four 32-byte big-endian draws at tape bytes [L, L + 128),
 *             L = zka_prove_tape_len(N, S) (a draw >= q gives ZKA_ERR_TAPE_RANGE); seeded calls draw t = 0..3 as rnd(q) on
 *             stream(seed, 4, t) (the rule of "Seeded randomness", domain 4)
 *   block     C1 = k g, C2 = x g + k Y, A0 = a g + beta h, A1 = c g, A2 = a g + c Y,
 *             e = SHA-256("ZKAttest/trace/v1" || params digest (32, "Hedged seeds") || Y || msg_hash || proof bytes
 *                 [0, HEAD_LEN) (R comS1 keyXcom keyYcom) || C1 || C2 || A0 || A1 || A2) big-endian mod q,
 *             s_x = a + e x, s_r = beta + e r, s_k = c + e k (mod q);  block = C1 C2 A0 A1 A2 s_x s_r s_k
 * Only rows the untraced call accepted get a block (proof_len grows by zka_trace_len()); a rejected row stays zeroed with
 * its status.  A trace point that is the war256 identity gives ZKA_ERR_IDENTITY_ENC.  With "self_check" on, every block is
 * also checked on the device and a row whose block fails gets ZKA_ERR_SELF_CHECK (counted in "self_check_fail").
 * Verify: a row shorter than the block, or whose block does not parse (points as the proof parser demands, scalars < q),
 * gives ZKA_ERR_MALFORMED (top precedence); otherwise the row gets the untraced verdict of its first proof_len -
 * zka_trace_len() bytes, and an accepted row also needs s_x g + s_r h = A0 + e keyXcom, s_k g = A1 + e C1 and
 * s_x g + s_k Y = A2 + e C2, or it gets ok = 0 with status 0.  The check is exact and uses no randomness.
 * Open: the block is parsed (ZKA_ERR_MALFORMED) and its relations checked (ZKA_ERR_TRACE_INVALID); the base proof is not
 * verified (verify first).  D = C2 - sk C1 = x g, and the row's index is the smallest j < N with (ring[j] mod q) g = D,
 * or 0xFFFFFFFF with ZKA_ERR_NOT_IN_RING.  Hashing the header binds a block to its proof's keyXcom, whose blinder is fresh.
 * Not covered: ring sets, hedged calls, the stand-alone sub-proofs, and a proof that an opening is correct.
 *
 * Pointers may be host or CUDA device pointers (detected per argument); host buffers are
 * staged through the library's stream.  The caller owns every buffer.
 * Return value: 0 on success, negative on a fatal (argument/CUDA) error — see zka_last_error.
 * Per-item `status[i]` mirrors the reference's throw sites (0 = ok).
 */
#ifndef ZKATTEST_H
#define ZKATTEST_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct zka_ctx zka_ctx;
typedef struct zka_params zka_params;
typedef struct zka_rings zka_rings;

enum {
  ZKA_OK = 0,
  ZKA_ERR_INVALID_PK = 1,        /* 'invalid public key' / 'point not in group'  zkpAttestList.ts:117, weier.ts:83 */
  ZKA_ERR_T_INFINITY = 2,        /* 'T[i] is at infinity'                        exp.ts:151 */
  ZKA_ERR_T1_INFINITY = 3,       /* 'T1 is at infinity'                          exp.ts:193 */
  ZKA_ERR_POINTS_DONT_ADD = 4,   /* "Points don't add up!"                       pointAdd.ts:105 */
  ZKA_ERR_TAPE_RANGE = 5,        /* a draw >= its modulus or tape too short (host must pre-filter) */
  ZKA_ERR_BAD_INDEX = 6,         /* `which` outside the ring */
  ZKA_ERR_IDENTITY_ENC = 7,      /* a P-256 proof point is the identity (1-byte encoding, weier.ts:247) */
  ZKA_ERR_R_INFINITY = 8,        /* 'R is at infinity'                           zkpAttestList.ts:159 */
  ZKA_ERR_MALFORMED = 9,         /* proof bytes do not parse (deserializePoint / deserializeScalar throw) */
  ZKA_ERR_PARAMS_NOT_FOUND = 10, /* exp.ts:270,302 */
  ZKA_ERR_SELF_CHECK = 11,       /* proof failed its self-check ("self_check" option, see "Self-checked proving") */
  ZKA_ERR_TRACE_INVALID = 12,    /* zka_open_batch: the trace block fails a relation under Y = sk g ("Traceable proofs") */
  ZKA_ERR_NOT_IN_RING = 13       /* zka_open_batch: the traced key is no entry of the ring */
};
/* Precedence: a row with several defects gets the code of the one the reference meets first.
 *   verify (zka_verify_batch*, zka_verify_exp_batch):  ZKA_ERR_MALFORMED (the whole proof is parsed first, so it wins over
 *     everything below), ZKA_ERR_R_INFINITY, a Groth-Kohlweiss draw out of range (ZKA_ERR_TAPE_RANGE); then a membership
 *     proof that fails gives ok = 0 with status 0, whatever the repetitions carry; then a generateIndices byte out of
 *     range (ZKA_ERR_TAPE_RANGE); then the sampled repetitions in sample order (generateIndices on the tape), the first
 *     one with a defect deciding: ZKA_ERR_PARAMS_NOT_FOUND, its first draw out of range, ZKA_ERR_T_INFINITY /
 *     ZKA_ERR_T1_INFINITY, its later draws out of range.
 *   prove: ZKA_ERR_INVALID_PK, ZKA_ERR_BAD_INDEX, then the repetitions in order; with the self-check on, a row that
 *     carries none of these is checked and may get ZKA_ERR_SELF_CHECK; a row that carries one keeps it unchecked. */

enum {
  ZKA_E_ARG = -1,     /* bad argument */
  ZKA_E_CUDA = -2,    /* CUDA runtime failure (no CPU fallback exists) */
  ZKA_E_NOMEM = -3
};

/* Create a context on CUDA device `device`.  Builds the fixed-base tables of the P-256 and
 * tomEdwards256 generators (instances.ts:22-54).  Fails (ZKA_E_CUDA) if no GPU is present. */
int zka_init(int device, zka_ctx** out);
void zka_shutdown(zka_ctx* ctx);
const char* zka_last_error(const zka_ctx* ctx);
int zka_version(void);
/* number of GPU kernels this context has launched so far (bench.py's gpu_launches) */
uint64_t zka_launch_count(const zka_ctx* ctx);

/* generateParamsList (zkpAttestList.ts:88-92, pedersen.ts:61-69): h_nist = G * rnd[0..32),
 * h_proof = g * rnd[32..64).  Draws must be < p256.n and < tom.order respectively. */
/* Which ProofGroup this library was built for, and the byte sizes of its points / scalars in the flat layout:
 *   libzkattest.so         "tomEdwards256"  67 / 33   (instances.ts:44-54, the default of generateParamsList)
 *   libzkattest_war256.so  "war256"         65 / 32   (instances.ts:34-41; the other legal SystemParametersList.ProofGroup,
 *                                                      zkpAttestList.ts:70) — same entry points, same grammar with these
 *                                                      sizes: wherever this header says 67 read point_bytes, 33 scalar_bytes.
 * A host picks the library by `params.ProofGroup.name`. */
int zka_proof_group(char* name, size_t cap, int* point_bytes, int* scalar_bytes);
int zka_params_generate(zka_ctx* ctx, const uint8_t rnd[64], uint8_t h_nist[65], uint8_t h_proof[67]);
/* SystemParametersList{NistGroup.h, ProofGroup.h, SecLevel} (zkpAttestList.ts:65-78) as a device
 * handle holding the fixed-base tables of both h points.  g is the curve generator. */
int zka_params_create(zka_ctx* ctx, const uint8_t h_nist[65], const uint8_t h_proof[67], uint32_t sec_level,
                      zka_params** out);
void zka_params_destroy(zka_params* params);

/* keyToInt (zkpAttestList.ts:94-102): x-coordinate of a raw P-256 key, 32 bytes big-endian.
 * status[i] = ZKA_ERR_INVALID_PK when pk[i] is not a point of the curve. */
int zka_key_to_int(zka_ctx* ctx, uint32_t count, const uint8_t* pk /*count x 65*/, uint8_t* x_out /*count x 32*/,
                   int32_t* status);

size_t zka_proof_max_len(uint32_t ring_size, uint32_t sec_level);
size_t zka_prove_tape_len(uint32_t ring_size, uint32_t sec_level);
size_t zka_verify_tape_len(uint32_t ring_size, uint32_t sec_level);

/* B independent proveSignatureList calls sharing one ring (zkpAttestList.ts:104-145). */
int zka_prove_batch(zka_ctx* ctx, const zka_params* params, uint32_t B,
                    const uint8_t* msg_hash /* B x 32 */, const uint8_t* sig /* B x 64, r||s */,
                    const uint8_t* pk /* B x 65 */, const uint32_t* which /* B */,
                    const uint8_t* ring /* N x 32 */, uint32_t N,
                    const uint8_t* tape /* B x tape_stride */, size_t tape_stride,
                    uint8_t* proofs /* B x proof_stride */, size_t proof_stride,
                    uint32_t* proof_len /* B */, int32_t* status /* B */);

/* B independent verifySignatureList calls sharing one ring (zkpAttestList.ts:147-184).
 * ok[i] = 1 iff the reference would return true.  The verifier tape holds, per proof, the
 * random relation scalars of Relation.drain (multimult.ts:168-173) and the 78 index draws of
 * generateIndices (exp.ts:95-109); layout in zk_verify.cuh.
 * Evaluation order (verdicts do not depend on it): a WEIGHTED sum over a chunk of proofs of the reference's three
 * linear combinations is checked first, as one wide-window MSM per group; each combination of each row is scaled by a
 * 128-bit weight from SHA-256 over the row's index in the call, ring index, message, tape row and the proof bytes the
 * verifier reads, so rows that share a tape row (or a seed), or a prover who knows the tape, cannot pick residuals that
 * cancel against the weights — the tape needs no property beyond the reference's own (limits: zk_verify_agg.cuh).
 * Only a chunk whose sum is not the identity — some proof wrong, rejected by the parsers, or (tomEdwards256, cofactor 4)
 * carrying a small-order component — is evaluated proof by proof with the reference's scalars (zka_stat). */
int zka_verify_batch(zka_ctx* ctx, const zka_params* params, uint32_t B,
                     const uint8_t* msg_hash /* B x 32 */, const uint8_t* ring /* N x 32 */, uint32_t N,
                     const uint8_t* proofs /* B x proof_stride */, size_t proof_stride,
                     const uint32_t* proof_len /* B */,
                     const uint8_t* tape /* B x tape_stride */, size_t tape_stride,
                     uint8_t* ok /* B */, int32_t* status /* B */);

/* The same with verifyExp's `secparam` (exp.ts:233-262) as a parameter: `samples` of the sec_level repetitions are
 * checked (verifySignatureList passes the literal 20, zkpAttestList.ts:177; the reference's own exp test passes
 * 80 on both sides).  The tape then holds 25 * samples packed exp drains: zka_verify_tape_len_ex. */
size_t zka_verify_tape_len_ex(uint32_t ring_size, uint32_t sec_level, uint32_t samples);
int zka_verify_batch_ex(zka_ctx* ctx, const zka_params* params, uint32_t B,
                        const uint8_t* msg_hash, const uint8_t* ring, uint32_t N,
                        const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                        const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status, uint32_t samples);

/* ---- seeded randomness (rule under "Seeded randomness" above): 32 bytes per proof instead of a tape ----
 * zka_prove_batch_seeded / zka_verify_batch_seeded: zka_prove_batch / zka_verify_batch_ex with the tape expanded on the
 * GPU from `seeds` (B x 32, host or device); every other argument, check and status is theirs.  Seeds count as the tape
 * does for the chunk schedule (host or device buffers) and the progress flags. */
int zka_prove_batch_seeded(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* msg_hash, const uint8_t* sig,
                           const uint8_t* pk, const uint32_t* which, const uint8_t* ring, uint32_t N,
                           const uint8_t* seeds /* B x 32 */, uint8_t* proofs, size_t proof_stride,
                           uint32_t* proof_len, int32_t* status);
int zka_verify_batch_seeded(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* msg_hash, const uint8_t* ring,
                            uint32_t N, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                            const uint8_t* seeds /* B x 32 */, uint32_t samples, uint8_t* ok, int32_t* status);
/* the tape a seed stands for: kind 0 = prover, all 3 + 44S + 5n draws (zka_prove_tape_len bytes); kind 1 = the verify
 * layout for `samples` (zka_verify_tape_len_ex bytes).  tape: B x tape_stride, host or device. */
int zka_seed_tape(zka_ctx* ctx, int kind, uint32_t B, const uint8_t* seeds, uint32_t ring_size, uint32_t sec_level,
                  uint32_t samples, uint8_t* tape, size_t tape_stride);

/* ---- ring sets: one batch against many key rings ----
 * The reference takes its own `keys` in every proveSignatureList / verifySignatureList call (zkpAttestList.ts:104-111,
 * 147-152); a ring set lets one batch do the same.  zka_rings_create: R >= 1 rings, ring r of sizes[r] entries in
 * [2, 2^20] (sizes: host memory); keys = the rings' 32-byte entries concatenated in ring order (host or device).  Each ring
 * is reduced mod the proof-group order and padded to 2^ceil(log2 sizes[r]) entries with ITS OWN first entry, exactly as
 * the ring of one zka_prove_batch call is (gk.ts:75-86).  ZKA_E_ARG when R = 0, a size is outside [2, 2^20] or the padded
 * rings hold more than 2^24 entries (512 MB).  The handle belongs to its context (like zka_params): destroy it first.
 *
 * zka_prove_batch_rings[_seeded] / zka_verify_batch_rings[_seeded] are zka_prove_batch[_seeded] / zka_verify_batch_ex /
 * zka_verify_batch_seeded with (ring, N) replaced by (rings, ring_of[B]): row i is proved / verified against ring
 * ring_of[i] (host or device), and its proof bytes, verdict and status are those of the one-ring call with that ring.
 *   - Per-row layout: each row's tape, seeded expansion, proof layout and status use its own ring size N_r and depth
 *     n_r = ceil(log2 N_r): 3 + 4S + 40Z + 5 n_r prover draws; the verify tape starts with 2 n_r + 1 GK drains.  Strides
 *     must cover the largest ring the call uses (zka_prove_tape_len, zka_verify_tape_len_ex, zka_proof_max_len of it).
 *   - which[i] >= N_r gives the row status ZKA_ERR_BAD_INDEX, also inside the padding (N_r = 5, which = 6).
 *   - Any ring_of[i] >= R: the call returns ZKA_E_ARG before any work.
 *   - The call is ONE pass of the batched pipeline whatever the order of ring depths in ring_of: its chunks are laid out for
 *     the largest depth the rows use and every row follows its own.  Rows in any order give the same bytes, and need no
 *     sorting or grouping to be fast.
 *   - The chunk schedule and the zka_set_progress flags are those of the one-ring call over the same B (zka_chunk_schedule). */
int zka_rings_create(zka_ctx* ctx, uint32_t R, const uint32_t* sizes /* R */, const uint8_t* keys /* sum(sizes) x 32 */,
                     zka_rings** out);
void zka_rings_destroy(zka_rings* rings);
int zka_prove_batch_rings(zka_ctx* ctx, const zka_params* params, const zka_rings* rings, const uint32_t* ring_of /* B */,
                          uint32_t B, const uint8_t* msg_hash, const uint8_t* sig, const uint8_t* pk, const uint32_t* which,
                          const uint8_t* tape, size_t tape_stride, uint8_t* proofs, size_t proof_stride, uint32_t* proof_len,
                          int32_t* status);
int zka_prove_batch_rings_seeded(zka_ctx* ctx, const zka_params* params, const zka_rings* rings, const uint32_t* ring_of,
                                 uint32_t B, const uint8_t* msg_hash, const uint8_t* sig, const uint8_t* pk, const uint32_t* which,
                                 const uint8_t* seeds /* B x 32 */, uint8_t* proofs, size_t proof_stride, uint32_t* proof_len,
                                 int32_t* status);
int zka_verify_batch_rings(zka_ctx* ctx, const zka_params* params, const zka_rings* rings, const uint32_t* ring_of, uint32_t B,
                           const uint8_t* msg_hash, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                           const uint8_t* tape, size_t tape_stride, uint32_t samples, uint8_t* ok, int32_t* status);
int zka_verify_batch_rings_seeded(zka_ctx* ctx, const zka_params* params, const zka_rings* rings, const uint32_t* ring_of,
                                  uint32_t B, const uint8_t* msg_hash, const uint8_t* proofs, size_t proof_stride,
                                  const uint32_t* proof_len, const uint8_t* seeds /* B x 32 */, uint32_t samples, uint8_t* ok,
                                  int32_t* status);

/* ---- hedged seeds (rule under "Hedged seeds" above) ----
 * zka_prove_batch_hedged / zka_prove_batch_rings_hedged: zka_prove_batch_seeded / zka_prove_batch_rings_seeded on the hedged
 * seed of every row instead of `seeds`; every other argument, check, status and the chunk schedule are theirs, except that
 * seeds may be NULL (deterministic proofs; the schedule then counts the seeds as device memory).  A ring-set row gets the
 * seed, and so the proof bytes, of the one-ring hedged call on its ring.
 * zka_hedge_seeds / zka_hedge_seeds_rings: the B x 32 seeds such a call derives, into `out` (host or device).  This is the
 * audit hook of the rule: ITS OUTPUT IS AS SECRET AS THE WITNESS. */
int zka_prove_batch_hedged(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* msg_hash, const uint8_t* sig,
                           const uint8_t* pk, const uint32_t* which, const uint8_t* ring, uint32_t N,
                           const uint8_t* seeds /* B x 32 or NULL */, uint8_t* proofs, size_t proof_stride,
                           uint32_t* proof_len, int32_t* status);
int zka_prove_batch_rings_hedged(zka_ctx* ctx, const zka_params* params, const zka_rings* rings, const uint32_t* ring_of,
                                 uint32_t B, const uint8_t* msg_hash, const uint8_t* sig, const uint8_t* pk, const uint32_t* which,
                                 const uint8_t* seeds /* B x 32 or NULL */, uint8_t* proofs, size_t proof_stride,
                                 uint32_t* proof_len, int32_t* status);
int zka_hedge_seeds(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* msg_hash, const uint8_t* sig,
                    const uint8_t* pk, const uint32_t* which, const uint8_t* ring, uint32_t N,
                    const uint8_t* seeds /* B x 32 or NULL */, uint8_t* out /* B x 32 */);
int zka_hedge_seeds_rings(zka_ctx* ctx, const zka_params* params, const zka_rings* rings, const uint32_t* ring_of, uint32_t B,
                          const uint8_t* msg_hash, const uint8_t* sig, const uint8_t* pk, const uint32_t* which,
                          const uint8_t* seeds /* B x 32 or NULL */, uint8_t* out /* B x 32 */);

/* ---- traceable proofs (rule under "Traceable proofs" above) ----
 * zka_trace_pubkey: Y = sk g (sk: 32 bytes big-endian in [1, q)).  zka_prove_batch_traced[_seeded]: the arguments of
 * zka_prove_batch[_seeded] plus Y; tape_stride must be >= zka_prove_tape_len(N, S) + 128 and proof_stride >=
 * zka_proof_max_len(N, S) + zka_trace_len().  zka_verify_batch_traced[_seeded]: the arguments of zka_verify_batch_ex /
 * zka_verify_batch_seeded plus Y.  zka_open_batch: sk, and per row the message hash the proof was made for (it is hashed
 * into e), the ring and the traced proofs; index[i] and status[i] per row.  A Y that does not parse as a point, or an sk of
 * 0 or >= q, gives ZKA_E_ARG.  Chunk schedule and progress flags are those of the untraced call (a flag is raised once
 * its chunk's blocks are in place). */
size_t zka_trace_len(void);
int zka_trace_pubkey(zka_ctx* ctx, const uint8_t sk[32], uint8_t* Y /* point_bytes */);
int zka_prove_batch_traced(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* msg_hash, const uint8_t* sig,
                           const uint8_t* pk, const uint32_t* which, const uint8_t* ring, uint32_t N, const uint8_t* tape,
                           size_t tape_stride, uint8_t* proofs, size_t proof_stride, uint32_t* proof_len, int32_t* status,
                           const uint8_t* Y);
int zka_prove_batch_traced_seeded(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* msg_hash,
                                  const uint8_t* sig, const uint8_t* pk, const uint32_t* which, const uint8_t* ring, uint32_t N,
                                  const uint8_t* seeds, uint8_t* proofs, size_t proof_stride, uint32_t* proof_len,
                                  int32_t* status, const uint8_t* Y);
int zka_verify_batch_traced(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* msg_hash, const uint8_t* ring,
                            uint32_t N, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                            const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status, uint32_t samples,
                            const uint8_t* Y);
int zka_verify_batch_traced_seeded(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* msg_hash,
                                   const uint8_t* ring, uint32_t N, const uint8_t* proofs, size_t proof_stride,
                                   const uint32_t* proof_len, const uint8_t* seeds, uint32_t samples, uint8_t* ok,
                                   int32_t* status, const uint8_t* Y);
int zka_open_batch(zka_ctx* ctx, const zka_params* params, const uint8_t sk[32], uint32_t B, const uint8_t* msg_hash /* B x 32 */,
                   const uint8_t* ring /* N x 32 */, uint32_t N, const uint8_t* proofs, size_t proof_stride,
                   const uint32_t* proof_len, uint32_t* index /* B */, int32_t* status /* B */);

/* ---- stand-alone sub-proof verifiers: the surface of the reference's own unit tests and benches ----
 * verifyExp(paramsNIST, paramsWario, Clambda, Px, Py, pi, secparam, Q?)   /root/reference/src/exp/exp.ts:233-349
 *   paramsNIST = (p256, g = base[i], h = NistGroup.h of `params`), paramsWario = ProofGroup of `params`;
 *   pi = the sec_level repetitions of `params` in the flat layout above (rep*), `samples` = secparam, q = NULL when
 *   the statement has no Q (test/exp/exp.test.ts:37-40) else B x 65 (65 zero bytes = identity).
 *   tape per statement: the sec_level-2 generateIndices bytes (exp.ts:101-106), zero-padded to 96 bytes, then the
 *   25 * samples packed Relation.drain scalars in consumption order (as in zka_verify_batch). */
int zka_verify_exp_batch(zka_ctx* ctx, const zka_params* params, uint32_t B,
                         const uint8_t* base /* B x 65 */, const uint8_t* com /* B x 65: Clambda */,
                         const uint8_t* px /* B x 67 */, const uint8_t* py /* B x 67 */, const uint8_t* q /* B x 65 or NULL */,
                         const uint8_t* proofs /* B x proof_stride */, size_t proof_stride, const uint32_t* proof_len /* B */,
                         const uint8_t* tape /* B x tape_stride */, size_t tape_stride, uint32_t samples,
                         uint8_t* ok /* B */, int32_t* status /* B */);
/* verifyMembership(params = ProofGroup, com, ring, proof)                /root/reference/src/proofGK/gk.ts:197-262
 *   proofs: GK blocks in the flat layout above; tape per statement: the 2n+1 Relation.drain scalars in call order
 *   (rel0_0, rel1_0, ..., relFinal), n = ceil(log2 N). */
int zka_verify_membership_batch(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* com /* B x 67 */,
                                const uint8_t* ring /* N x 32 */, uint32_t N,
                                const uint8_t* proofs /* B x proof_stride */, size_t proof_stride, const uint32_t* proof_len /* B */,
                                const uint8_t* tape /* B x tape_stride */, size_t tape_stride,
                                uint8_t* ok /* B */, int32_t* status /* B */);

/* verifyEquality(params, C1, C2, pi)            /root/reference/src/commit/equality.ts:80-116   points: B x 2 x 67
 * verifyMult(params, Cx, Cy, Cz, pi)             /root/reference/src/commit/mult.ts:133-175      points: B x 3 x 67
 * verifyPointAdd(params, PX,PY,QX,QY,RX,RY, pi)  /root/reference/src/exp/pointAdd.ts:181-259     points: B x 6 x 67
 * over params = ProofGroup; proofs: B x 233 / 633 / 3266 bytes in the flat layout above; tape per statement: the 2 / 5 /
 * 24 Relation.drain scalars (mod tomEdwards256.order) in call order. */
int zka_verify_equality_batch(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* points, const uint8_t* proofs,
                              const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status);
int zka_verify_mult_batch(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* points, const uint8_t* proofs,
                          const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status);
int zka_verify_pointadd_batch(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* points, const uint8_t* proofs,
                              const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status);

/* ---- stand-alone sub-proof provers ----
 * proveExp(paramsNIST = (p256, base[i], NistGroup.h), paramsWario = ProofGroup, s, Cs, P = pk, Px, Py, sec_level, Q?)
 *                                                                          /root/reference/src/exp/exp.ts:126-231
 *   The statement is s*base - Q = pk (Q = NULL: s*base = pk, as in test/exp/exp.test.ts:26-38); it is checked and
 *   ZKA_ERR_POINTS_DONT_ADD reported otherwise (pointAdd.ts:104).  Tape: the layout of zka_prove_batch — draws 0..2 are
 *   the blinders of Cs, Px, Py (drawn when those commitments were made: Cs = s*base + r0*h, Px = commit(pk.x, r1),
 *   Py = commit(pk.y, r2)), then 4 per repetition, then 40 per 0-bit repetition.  Rows: the repetitions only
 *   (proof_stride >= sec_level * 3596), as consumed by zka_verify_exp_batch. */
int zka_prove_exp_batch(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* base /* B x 65 */,
                        const uint8_t* s /* B x 32 */, const uint8_t* pk /* B x 65 */, const uint8_t* q /* B x 65 or NULL */,
                        const uint8_t* tape, size_t tape_stride, uint8_t* proofs, size_t proof_stride,
                        uint32_t* proof_len /* B */, int32_t* status /* B */);
/* proveMembership(params = ProofGroup, com, index, ring)                    /root/reference/src/proofGK/gk.ts:94-195
 *   com_r: blinder of com = commit(ring[index]); tape: the 5n draws r_i, a_i, s_i, t_i, rho_i per round (gk.ts:117-123).
 *   Rows: the GK block (proof_stride >= 1 + 4n*67 + (3n+1)*33). */
int zka_prove_membership_batch(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* com_r /* B x 32 */,
                               const uint32_t* index /* B */, const uint8_t* ring /* N x 32 */, uint32_t N,
                               const uint8_t* tape, size_t tape_stride, uint8_t* proofs, size_t proof_stride,
                               uint32_t* proof_len /* B */, int32_t* status /* B */);

/* proveEquality(params, x, C1, C2)          /root/reference/src/commit/equality.ts:60-78
 *   scalars: B x [x, C1.r, C2.r] (32 bytes each);  tape: k, A1.r, A2.r;  out: C1 C2 (B x 2 x 67), proofs B x 233
 * proveMult(params, x, y, z, Cx, Cy, Cz)     /root/reference/src/commit/mult.ts:93-131
 *   scalars: B x [x, y, z, Cx.r, Cy.r, Cz.r];      tape: k_x k_y k_z Ax.r Ay.r Az.r A4_1.r;  out: Cx Cy Cz, proofs B x 633
 * provePointAdd(params, P, Q, R, PX, PY, QX, QY, RX, RY)   /root/reference/src/exp/pointAdd.ts:92-163
 *   points: B x [P, Q, R] (65 bytes each, P + Q = R on P-256);  blinders: B x [PX.r PY.r QX.r QY.r RX.r RY.r];
 *   tape: the 38 draws of SURVEY.md 3.1 (C8.r C10.r C11.r C13.r, pi8[7], pi10[7], pi11[7], pix[3], pi13[7], piy[3]);
 *   out: the six coordinate commitments (B x 6 x 67), proofs B x 3266.
 * The statement's commitments are given by their openings (the prover knows them); the library returns their points. */
int zka_prove_equality_batch(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* scalars, const uint8_t* tape,
                             size_t tape_stride, uint8_t* commitments, uint8_t* proofs, int32_t* status);
int zka_prove_mult_batch(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* scalars, const uint8_t* tape,
                         size_t tape_stride, uint8_t* commitments, uint8_t* proofs, int32_t* status);
int zka_prove_pointadd_batch(zka_ctx* ctx, const zka_params* params, uint32_t B, const uint8_t* points, const uint8_t* blinders,
                             const uint8_t* tape, size_t tape_stride, uint8_t* commitments, uint8_t* proofs, int32_t* status);

/* ---- measurement hooks (bench.py) ----
 * zka_get_stream: the cudaStream_t every kernel of this context is launched on (so callers can
 * record CUDA events on the launching stream).  zka_set_profiling(1) brackets every launch with a
 * CUDA-event pair; zka_profile_json writes {"<task>": {"launches":n,"ms":t,"items":k}, ...}. */
void* zka_get_stream(zka_ctx* ctx);
int zka_set_profiling(zka_ctx* ctx, int enable);
int zka_profile_reset(zka_ctx* ctx);
size_t zka_profile_json(zka_ctx* ctx, char* buf, size_t cap);
/* tuning knobs read at zka_init from the environment (zka_config reports the first three):
 *   ZKA_TOM_NWIN    lookups per scalar of the tomEdwards256 fixed-base tables g and h, 11..128, default 11.  The 257 bits
 *                   of a walk (256 of the scalar, 1 carry of the signed recoding) are cut into windows of
 *                   w = floor(257 / n) bits and, on top of them, 257 - w n windows of w + 1 bits; a window of b bits holds
 *                   2^(b-1) + 1 entries of 128 B.  11: 7 windows of 23 bits + 4 of 24 = 8.05 GB per base; 12: 7 of 21 + 5
 *                   of 22 = 2.3 GB; 16: 15 of 16 + 1 of 17 = 71 MB.  If the tables do not fit in the device's free memory
 *                   at zka_init, the context walks one lookup more (12 for the default) and says so: zka_config reports
 *                   the shape in use, zka_stat "tom_fallback" is 1.
 *   ZKA_TOM_W       instead: the same width for all windows, 2..24 ((256 + w) / w windows of 2^(w-1) + 1 entries: 3.2 GB
 *                   per base at 22, 12 lookups; 11.8 GB at 24, 11 lookups).  Takes precedence; never replaced by a
 *                   smaller table.  The only form the war256 build knows (default 22).
 *   ZKA_TOM_TABLE_MAX  bytes: a tomEdwards256 table larger than this is treated as an allocation that failed
 *   ZKA_P256_HW     window bits of the P-256 G / NistGroup.h tables, 8..24, default 20 (872 MB per base)
 *   ZKA_CHUNK       largest chunk (proofs per pipeline pass) when all buffers are device memory, default 4096
 *   ZKA_HOST_CHUNK  largest chunk when buffers are host memory, default 2048; the schedule is tapered
 *                   (quarter, half, full ..., half, quarter chunks) so that little copy time is exposed before
 *                   the first and after the last kernel
 *   ZKA_LANES       concurrent pipelines inside one prove / verify call, 1..8, default 3: the batch is cut
 *                   into chunks dealt round-robin to the lanes; every lane has its own streams and workspace
 *                   and (beyond the first) its own host thread for the duration of the call, so the
 *                   latency-bound stages and the host<->device copies of one chunk overlap the
 *                   multiplier-bound kernels of another
 *   ZKA_TAPE_SPLIT  1 (default): a host tape travels in two strided copies — the 3 + 4 S draws before the challenge, then
 *                   the item / GK draws up to the longest proof of the chunk; 0: one full-stride copy up front
 *   ZKA_AGG, ZKA_AGG_C   the verifier's chunk-wide aggregate check (see zka_stat): 0 disables it / window bits 4..16
 *   ZKA_TRACE       per-chunk timeline of the host-buffer pipelines on stderr (adds synchronisations) */
int zka_config(const zka_ctx* ctx, int* tom_w, int* tom_nwin, int* chunk);
int zka_lanes(const zka_ctx* ctx);
/* change a knob between calls: key in {"lanes", "chunk", "host_chunk", "agg" (1 = off, 2 = on), "agg_c" (4..16),
 * "self_check" (1 = off, the default; 2 = on: see "Self-checked proving")}, value >= 1 */
int zka_set_option(zka_ctx* ctx, const char* key, long value);
/* counters since zka_init: "agg_pass" = verifier chunks accepted as a whole by the chunk-wide aggregate check (the
 * sum over all proofs of the chunk of the reference's three linear combinations, multimult.ts:147-174, evaluated as one
 * wide-window MSM; every relation carries its own random scalar, so the sum is the identity iff (w.h.p.) every
 * per-proof combination is), "agg_fail" = chunks that went on to the per-proof evaluation (some proof invalid or
 * already rejected by the parsers; verdicts and statuses are then exactly the per-proof ones); both count verify calls
 * only, not the chunks of the prover's self-check.  "self_check_rows" = rows the self-check verified, "self_check_fail" =
 * rows it gave ZKA_ERR_SELF_CHECK.  Not counters:
 * "tom_n_lo" = how many of the tom_nwin windows zka_config reports have tom_w bits (the others have tom_w + 1),
 * "tom_fallback" = 1 when the tables asked for did not fit and the context walks one lookup more.  -1: unknown key.
 * ZKA_AGG=0 disables the aggregate check, ZKA_AGG_C=4..16 fixes its window bits. */
long long zka_stat(zka_ctx* ctx, const char* key);

/* Progress of a running zka_prove_batch (another host thread may watch it): the call cuts its batch into the chunks of
 * zka_chunk_schedule (off[0..n], deterministic for a given B, kind of buffers and knobs — the same on every rank); flags[k]
 * becomes 1 (written by a CUDA host callback) when the proofs of rows [off[k], off[k+1]) are complete in the caller's
 * DEVICE buffers.  bench.py uses it to queue the all-gather of finished chunks, in chunk order, while later chunks are
 * still being proved.  zka_set_progress(ctx, NULL, 0) switches it off. */
int zka_set_progress(zka_ctx* ctx, volatile uint32_t* flags, uint32_t cap);
int zka_chunk_schedule(zka_ctx* ctx, uint32_t B, int host_buffers, uint32_t* off /* cap entries */, uint32_t cap);

/* ---- multi-GPU helpers (SURVEY.md 8(e)): a rank's proofs as ONE contiguous block for the NCCL all-gather.
 * Proof b starts at offsets[b] = sum_{i<b} align16(proof_len[i]); offsets[B] is the block length (the caller
 * checks offsets[B] <= cap; pieces that would cross `cap` are not written).  Device pointers only.  With a
 * non-NULL `stream` (a cudaStream_t) the two kernels are enqueued there and the call returns without waiting;
 * with NULL they run on the library's stream and the call waits for them.
 * 16-byte aligned rows (proof_stride % 16 == 0, aligned base pointers) are moved with 16-byte accesses. */
int zka_proofs_pack(zka_ctx* ctx, uint32_t B, const uint8_t* proofs /* B x proof_stride */, size_t proof_stride,
                    const uint32_t* proof_len /* B */, uint8_t* packed, size_t cap, uint64_t* offsets /* B + 1 */,
                    void* stream);
int zka_proofs_unpack(zka_ctx* ctx, uint32_t B, const uint8_t* packed, size_t cap, const uint32_t* proof_len /* B */,
                      uint8_t* proofs /* B x proof_stride */, size_t proof_stride, uint64_t* offsets /* B + 1 */,
                      void* stream);

/* ---- layer-wise entry points (parity tests of the arithmetic underneath) ---- */
/* Pedersen commit in the proof group: out[i] = v[i]*g + r[i]*h  (pedersen.ts:53-58 with r given) */
int zka_tom_commit_batch(zka_ctx* ctx, const zka_params* params, uint32_t count,
                         const uint8_t* v /* count x 32 */, const uint8_t* r /* count x 32 */,
                         uint8_t* out /* count x 67 */);
/* P-256 scalar multiplication out[i] = k[i] * base[i] (Point.mul, group.ts:133-152);
 * base == NULL means the generator.  Identity result is encoded as 65 zero bytes. */
int zka_p256_mul_batch(zka_ctx* ctx, uint32_t count, const uint8_t* base /* count x 65 or NULL */,
                       const uint8_t* k /* count x 32 */, uint8_t* out /* count x 65 */);
/* field arithmetic: field 0 = p256.p (= tom.order), 1 = p256.n, 2 = tom.p (33-byte operands);
 * op 0 = a*b, 1 = a+b, 2 = a-b, 3 = a^-1 (0 -> 0; binary almost-inverse), 4 = a^(p-2) (Fermat ladder, the
 * cross-check of op 3).  Operands/results big-endian, canonical. */
int zka_field_op_batch(zka_ctx* ctx, int field, int op, uint32_t count, const uint8_t* a, const uint8_t* b,
                       uint8_t* out);
/* hashPoints (group.ts:221-233): 80-bit challenge (10 bytes) of `len[i]` message bytes each */
int zka_hash80_batch(zka_ctx* ctx, uint32_t count, const uint8_t* msgs, size_t msg_stride, const uint32_t* len,
                     uint8_t* out /* count x 10 */);

#ifdef __cplusplus
}
#endif
#endif /* ZKATTEST_H */
