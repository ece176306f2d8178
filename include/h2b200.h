/* h2b200.h — C ABI of libh2b200: the sm_90a back end for the create_proof hot path of halo2-lib
 * (multi-scalar multiplication over BN254 G1, NTT over BN254 Fr, column-wise witness assignment).
 *
 * This is the surface a `halo2_proofs`-compatible Rust crate binds with `extern "C"` in place of the rayon
 * CPU code; halo2-lib selects that crate through its own plug point, the `cuda` feature alias
 *     halo2-base/src/lib.rs:25-28   (#[cfg(feature = "cuda")] pub use halo2_proofs_axiom_gpu as halo2_proofs;)
 * so GateInstructions / RangeInstructions / FpChip / EccChip circuits and the keygen_pk / create_proof
 * entry points (sole call site halo2-base/src/utils/testing.rs:40-48) are untouched.  INTEGRATION.md shows
 * the Rust-side binding.
 *
 * Conventions
 *  - Field element  = uint64_t[4], little-endian limbs, Montgomery form (R = 2^256): the `[u64;4]` contract
 *    of halo2-base/src/utils/mod.rs:332-377 and the in-memory layout of halo2curves bn256::{Fr,Fq}.
 *  - G1Affine       = x||y (8 limbs), identity = (0,0).   G1 (Jacobian) = x||y||z (12 limbs), identity z = 0.
 *  - Every function returns an int status: 0 = OK, negative = error class below; the message is available
 *    from h2b_last_error().  No C++ exception and no abort crosses this boundary (Rust `panic = unwind`,
 *    reference Cargo.toml:31; unwinding through extern "C" is UB).
 *  - Host-pointer entry points own no caller memory: buffers are read/written during the call only.
 *    `_dev` entry points take device pointers (same layouts) and enqueue on the context's stream without
 *    synchronising; the caller owns those allocations (e.g. torch tensors) and the synchronisation.
 *    Exceptions, all on the host side only (results are stream-ordered either way): a call that needs a larger scratch
 *    workspace than any call before it on this context waits for the device once (the workspaces are grow-only);
 *    h2b_quotient_graph_dev / h2b_permutation_fold_dev / h2b_lookup_fold_dev / h2b_poly_lincomb_dev copy a table of a few
 *    hundred bytes from pageable host memory, which the CUDA runtime stages before returning (not capturable into a CUDA
 *    graph); h2b_assign_columns_dev with more than 64 columns waits for its pinned span block; the first transform of a
 *    new domain size builds its twiddle plan and waits for it; h2b_permute_expression_pair_dev and the calls that return
 *    a value to the host (h2b_eval_polynomial*_dev, h2b_poly_download, h2b_profile_*) synchronise the stream.
 *  - A context is bound to ONE device (one process per GPU); calls on one context are serialised by an
 *    internal mutex, so the library is re-entrant from rayon worker threads
 *    (halo2-base/src/gates/flex_gate/threads/parallelize.rs:8-29 runs user code on many threads).
 *  - There is no CPU fallback: without a CUDA device h2b_ctx_create fails with H2B_ERR_CUDA.
 */
#ifndef H2B200_H
#define H2B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define H2B_OK 0
#define H2B_ERR_ARG (-1)   /* bad argument (null pointer, size mismatch, k out of range) */
#define H2B_ERR_CUDA (-2)  /* CUDA runtime error (message carries cudaGetErrorString) */
#define H2B_ERR_OOM (-3)   /* device or host allocation failed */
#define H2B_ERR_LAYOUT (-4) /* witness layout error: where the Rust code panics (out of columns / rows) */
#define H2B_ERR_UNSATISFIED (-5) /* plonk::Error::ConstraintSystemFailure: a lookup input is not in the table */

typedef struct h2b_ctx h2b_ctx;
typedef struct h2b_srs h2b_srs;

#define H2B_BASIS_MONOMIAL 0 /* ParamsKZG::g          -> ParamsKZG::commit          */
#define H2B_BASIS_LAGRANGE 1 /* ParamsKZG::g_lagrange -> ParamsKZG::commit_lagrange */

/* ---- context -------------------------------------------------------------------------------------- */
int h2b_ctx_create(int device, h2b_ctx** out);
/* One process, n_dev GPUs (the reference's create_proof is ONE in-process call, halo2-base/src/utils/testing.rs:40-48): the
 * handle is an ordinary context on dev_ids[0] that also drives the other devices.  On such a context
 *   h2b_srs_upload                      shards the bases over the devices by contiguous index range (resident per device),
 *   h2b_msm_g1 / h2b_msm_g1_batch       commit every shard on its own device and return the FULL sums: the partial sums meet
 *                                       in the fused all-reduce kernel over in-process peer mappings (no IPC, no NCCL),
 *   h2b_*_batch transforms              deal polynomial j to device j mod n_dev, all devices pipelined concurrently,
 * and every other entry point (assignment, `_dev` calls, ...) runs on dev_ids[0].  SRS handles of a group are only valid
 * on that group.  h2b_ctx_device_count returns n_dev (1 for h2b_ctx_create). */
int h2b_ctx_create_multi(const int* dev_ids, int n_dev, h2b_ctx** out);
int h2b_ctx_device_count(const h2b_ctx* ctx);
void h2b_ctx_destroy(h2b_ctx* ctx);
/* Use a caller-owned cudaStream_t (e.g. torch.cuda.current_stream().cuda_stream) for all work; NULL = the
 * context's own stream. */
int h2b_ctx_set_stream(h2b_ctx* ctx, void* cuda_stream);
int h2b_ctx_synchronize(h2b_ctx* ctx);
/* A second in-order queue of the same context: between h2b_ctx_side_begin and h2b_ctx_side_end every `_dev` call is
 * enqueued on the context's side stream, which first waits for everything enqueued so far on the main stream;
 * h2b_ctx_side_join makes the main stream wait for the side work enqueued so far.  The resident prover runs the
 * lagrange_to_coeff / coeff_to_extended of the columns that already exist beside the next phase's commitments this way.
 * The side queue has its own scratch workspaces; the caller keeps the two queues on disjoint polynomials, and must not run
 * a batched MSM (which uses all workspace sets) on the main queue while side work that is not a transform is in flight. */
int h2b_ctx_side_begin(h2b_ctx* ctx);
int h2b_ctx_side_end(h2b_ctx* ctx);
int h2b_ctx_side_join(h2b_ctx* ctx);
/* Tuning switches (results never depend on them).  Keys:
 *   "ntt.max_ctas_per_sm" 0 (default: as many as fit), 1 or 2: the transforms of this context leave room on every SM — for a
 *                        transform that runs in the background of a latency-bound MSM pipeline (small multi-GPU shards)
 *   "msm.batch_group"    1..16 (0 = default, chosen from the domain size): how many MSMs of one batch call share a single
 *                        sort / accumulate / bucket-reduction pipeline (1 = every MSM runs its own, on one of three lanes)
 * and one switch that selects between two equally valid outputs (see h2b_permute_expression_pair):
 *   "lookup.leftover_order"  0 (default): left-over table values fill the repeated rows front to back; 1: from the back */
int h2b_ctx_set_option(h2b_ctx* ctx, const char* key, int64_t value);
/* Last error message of this context (or of the failed h2b_ctx_create when ctx == NULL). */
const char* h2b_last_error(const h2b_ctx* ctx);
/* Number of kernels this context has launched so far (bench.py's `gpu_launches`). */
uint64_t h2b_kernel_launches(const h2b_ctx* ctx);
const char* h2b_version(void);
/* Device-side timing of the library's own kernels (CUDA events on the launching stream): `filter` is a
 * substring of the kernel name ("k_accumulate"), "*" for all, NULL/"" to switch off.  h2b_profile_read
 * synchronises the stream and returns the summed duration and count of the matching launches since the
 * last h2b_profile_reset.  Used by bench.py for the roofline of the dominant kernel. */
int h2b_profile_enable(h2b_ctx* ctx, const char* filter);
int h2b_profile_reset(h2b_ctx* ctx);
int h2b_profile_read(h2b_ctx* ctx, const char* kernel, double* total_ms, uint64_t* launches);
/* Appends one CSV line per recorded launch to `path`: kernel, stream, start_us, end_us after the caller's CUDA event
 * `origin` (cudaEvent_t with timing).  Synchronises the device.  A timeline tool, not a product call. */
int h2b_profile_dump(h2b_ctx* ctx, void* origin_cuda_event, const char* path);

/* ---- SRS: replaces the base arrays of ParamsKZG<Bn256> (halo2-base/src/utils/mod.rs:401-443) ------- */
/* Uploads this device's shard [begin, begin+count) of the 2^k monomial bases `g` and Lagrange bases
 * `g_lagrange` (each 2^k x 8 limbs on the host; either may be NULL) and builds the per-window multiples
 * 2^(c*w) * P_i the fixed-base MSM consumes.  Single GPU: begin = 0, count = 2^k. */
int h2b_srs_upload(h2b_ctx* ctx, const uint64_t* g, const uint64_t* g_lagrange, uint32_t k, size_t begin,
                   size_t count, h2b_srs** out);
/* Same, bases already on the device (count x 8 limbs each, the shard only). */
int h2b_srs_upload_dev(h2b_ctx* ctx, const void* d_g, const void* d_g_lagrange, uint32_t k, size_t begin,
                       size_t count, h2b_srs** out);
/* Window size c (bits) and number of table levels W = ceil(255 / c) chosen for this shard. */
int h2b_srs_info(const h2b_srs* srs, int* window_bits, int* windows);
void h2b_srs_destroy(h2b_ctx* ctx, h2b_srs* srs);

/* Keygen-side SRS utilities (SURVEY.md §8(f) rank 3; halo2-axiom 0.5.3 poly/kzg/commitment.rs, not vendored — restated).
 * h2b_g_to_lagrange: `g_to_lagrange(g_projective, k)`: g_lagrange[i] = 2^-k * sum_j omega^(-i j) g[j] (a radix-2 FFT over
 * G1), normalised to affine; g, g_lagrange: 2^k x 8 limbs.
 * h2b_srs_setup: `ParamsKZG::setup` for a caller-supplied tau (the reference draws it from ChaCha20Rng seed 0,
 * halo2-base/src/utils/mod.rs:439-443 — that draw stays on the Rust side): g[i] = tau^i * base, g_lagrange[i] =
 * L_i(tau) * base; either output may be NULL.  tau must not be a 2^k-th root of unity.
 * h2b_g1_check_on_curve: counts the points that are neither (0,0) nor on y^2 = x^3 + 3 (what `ParamsKZG::read` must
 * reject, utils/mod.rs:401-424).
 * h2b_params_raw_view: offsets into a `ParamsKZG::write` image in SerdeFormat::RawBytes — u32 LE k, 2^k x 64 B g,
 * 2^k x 64 B g_lagrange, 128 B g2, 128 B s_g2, all Montgomery limbs, i.e. exactly the layouts of this header, so the
 * file can be uploaded with h2b_srs_upload without a copy.  Host-only, no device work. */
int h2b_g_to_lagrange(h2b_ctx* ctx, const uint64_t* g, uint32_t k, uint64_t* g_lagrange);
int h2b_g_to_lagrange_dev(h2b_ctx* ctx, const void* d_g, uint32_t k, void* d_g_lagrange);
int h2b_srs_setup(h2b_ctx* ctx, const uint64_t tau[4], const uint64_t base_xy[8], uint32_t k, uint64_t* g, uint64_t* g_lagrange);
int h2b_srs_setup_dev(h2b_ctx* ctx, const uint64_t tau[4], const uint64_t base_xy[8], uint32_t k, void* d_g, void* d_g_lagrange);
int h2b_g1_check_on_curve(h2b_ctx* ctx, const uint64_t* points_xy, size_t n, size_t* off_curve);
int h2b_g1_check_on_curve_dev(h2b_ctx* ctx, const void* d_points_xy, size_t n, size_t* off_curve);
int h2b_params_raw_view(const uint8_t* bytes, size_t len, uint32_t* k, size_t* g_offset, size_t* g_lagrange_offset,
                        size_t* g2_offset, size_t* s_g2_offset);
/* SerdeFormat::Processed (what `ParamsKZG::write` emits by default and `gen_srs` caches as ./params/kzg_bn254_{k}.srs,
 * halo2-base/src/utils/mod.rs:413-435): compressed G1 = 32 bytes, x little-endian, bit 7 of the last byte = point at
 * infinity, bit 6 = parity of y.  h2b_g1_decompress: n encodings -> n affine points (Montgomery, identity (0,0)) through a
 * square root in Fq per point; *invalid = encodings that are no point (x >= p, x^3 + 3 a non-residue, bad flags; their
 * output is (0,0)).  h2b_params_processed_view: offsets of the image (u32 LE k, 2^k x 32 B g, 2^k x 32 B g_lagrange,
 * 64 B g2, 64 B s_g2).  h2b_srs_read_processed: the device side of `ParamsKZG::read` — decompress the shard
 * [begin, begin + count) (count = 0: everything) of both bases and build the SRS handle; H2B_ERR_ARG if the image is
 * malformed or holds an invalid encoding. */
#define H2B_G1_FLAG_IDENTITY 128u /* the flag bits of byte 31 of a compressed G1 point */
#define H2B_G1_FLAG_Y_ODD 64u
int h2b_g1_decompress(h2b_ctx* ctx, const uint8_t* bytes, size_t n, uint64_t* out_xy, size_t* invalid);
int h2b_g1_decompress_dev(h2b_ctx* ctx, const void* d_bytes, size_t n, void* d_out_xy, size_t* invalid);
int h2b_params_processed_view(const uint8_t* bytes, size_t len, uint32_t* k, size_t* g_offset, size_t* g_lagrange_offset,
                              size_t* g2_offset, size_t* s_g2_offset);
int h2b_srs_read_processed(h2b_ctx* ctx, const uint8_t* bytes, size_t len, size_t begin, size_t count, h2b_srs** out);
/* The write side (`gen_srs` = read_or_create_srs, halo2-base/src/utils/mod.rs:413-443, and `ParamsKZG::write`).
 * h2b_g1_compress: n affine points (Montgomery, identity (0,0)) -> n x 32-byte encodings, the exact inverse of
 * h2b_g1_decompress (canonical x little-endian, bit 6 of byte 31 = parity of the canonical y, identity = all zero but bit 7
 * of byte 31); one thread per point.
 * h2b_srs_seeded_tau: the tau of `ParamsKZG::setup(k, ChaCha20Rng::from_seed(seed))` (gen_srs: seed = 32 zero bytes):
 * rand_chacha's ChaCha20 stream (64-bit block counter from 0, stream 0), 64 bytes through `Fr::random` =
 * from_uniform_bytes, (lo + hi 2^256) mod r; tau in Montgomery form.  Host-only.
 * h2b_g2_generator_mul: g2 = the EIP-197 generator of the BN254 twist and s_g2 = tau * g2 in both encodings of a params
 * image: processed = g2 | s_g2 compressed (64 bytes each: x.c0 | x.c1 canonical little-endian, bit 7 of byte 63 =
 * identity, bit 6 = sgn0(y)), raw = g2 | s_g2 as x.c0 | x.c1 | y.c0 | y.c1 Montgomery limbs (128 bytes each); either output may
 * be NULL.  tau must be below r.  Host-only.
 * h2b_params_write_processed / h2b_params_write_raw: the image u32 LE k | g | g_lagrange | g2 | s_g2 from the device bases
 * d_g, d_g_lagrange (2^k x 8 limbs each) and the G2 pair of h2b_g2_generator_mul, into the caller's buffer `out`: *len is
 * its capacity on entry and the image size on return; out = NULL only asks for the size.  Processed compresses both bases on
 * the device into one staging buffer and downloads it with one copy.  h2b_params_processed_view / h2b_srs_read_processed /
 * h2b_params_raw_view read the images back. */
int h2b_g1_compress(h2b_ctx* ctx, const uint64_t* xy, size_t n, uint8_t* bytes);
int h2b_g1_compress_dev(h2b_ctx* ctx, const void* d_xy, size_t n, void* d_bytes);
int h2b_srs_seeded_tau(const uint8_t seed[32], uint64_t tau[4]);
int h2b_g2_generator_mul(const uint64_t tau[4], uint8_t processed[128], uint8_t raw[256]);
int h2b_params_write_processed(h2b_ctx* ctx, const void* d_g, const void* d_g_lagrange, uint32_t k, const uint8_t g2[128], uint8_t* out,
                               size_t* len);
int h2b_params_write_raw(h2b_ctx* ctx, const void* d_g, const void* d_g_lagrange, uint32_t k, const uint8_t g2[256], uint8_t* out,
                         size_t* len);

/* ---- MSM: replaces halo2curves-axiom 0.7.3 msm::best_multiexp(coeffs, bases) -> G1, as reached from
 *      ParamsKZG::commit / commit_lagrange inside create_proof (SURVEY.md §3.3, §8 a2/a4) ------------- */
/* out = sum_{i in shard} scalars[i] * basis[i].  `scalars` holds the `n` scalars of THIS shard
 * (n == count of the SRS).  Result: a valid Jacobian representative (not normalised), like best_multiexp. */
int h2b_msm_g1(h2b_ctx* ctx, const h2b_srs* srs, int basis, const uint64_t* scalars, size_t n,
               uint64_t out_xyz[12]);
/* m independent commitments of one prover phase (all advice columns, the lookup permuted pair, the h(X) pieces,
 * ...): basis[j] selects the basis of column j, scalars[j] points at its n scalars; out = m x 12 limbs.  Uploads
 * are pipelined against the kernels and the MSMs are spread over the context's lanes (see h2b_msm_g1_batch_dev). */
int h2b_msm_g1_batch(h2b_ctx* ctx, const h2b_srs* srs, const int* basis, const uint64_t* const* scalars, size_t m,
                     size_t n, uint64_t* out_xyz);
/* Same as h2b_msm_g1_batch, but when the context's NVLink mailboxes are connected (h2b_peer_connect) the m partial
 * sums of all GPUs are combined on the device by the fused all-reduce kernel before the single device-to-host copy:
 * out = the m FULL commitments on every rank.  Without peers it is h2b_msm_g1_batch. */
int h2b_msm_g1_batch_reduced(h2b_ctx* ctx, const h2b_srs* srs, const int* basis, const uint64_t* const* scalars, size_t m,
                             size_t n, uint64_t* out_xyz);
/* Ad-hoc bases (n x 8 limbs on the host), no precomputation. */
int h2b_msm_g1_bases(h2b_ctx* ctx, const uint64_t* bases, const uint64_t* scalars, size_t n,
                     uint64_t out_xyz[12]);
/* Device-resident variants: d_scalars = n x 4 limbs, d_out = 12 limbs, all on the device; asynchronous. */
int h2b_msm_g1_dev(h2b_ctx* ctx, const h2b_srs* srs, int basis, const void* d_scalars, size_t n, void* d_out);
int h2b_msm_g1_bases_dev(h2b_ctx* ctx, const void* d_bases, const void* d_scalars, size_t n, void* d_out);
/* m device-resident columns (basis[j] per column); the MSMs are spread over the context's internal lanes
 * (streams + workspaces) so that the latency-bound bucket reduction of one overlaps the bucket accumulation
 * of the next, and joined back onto the context's stream.  d_scalars = host array of m device pointers;
 * d_out = m x 12 limbs on the device. */
int h2b_msm_g1_batch_dev(h2b_ctx* ctx, const h2b_srs* srs, const int* basis, const void* const* d_scalars, size_t m,
                         size_t n, void* d_out);
/* out = sum of m Jacobian points (host, m x 12 limbs): combines the per-GPU partial sums after the
 * all-gather (EC addition is not an NCCL reduction op).  Runs on the device. */
int h2b_g1_sum(h2b_ctx* ctx, const uint64_t* points_xyz, size_t m, uint64_t out_xyz[12]);
int h2b_g1_sum_dev(h2b_ctx* ctx, const void* d_points_xyz, size_t m, void* d_out);
/* Batch-normalise m Jacobian points to affine-normalised form (x, y, R) / identity (0, R, 0), in place. */
int h2b_g1_normalize(h2b_ctx* ctx, uint64_t* points_xyz, size_t m);
/* out[i] = scalars[i] * base (affine, n x 8 limbs): the per-point work of ParamsKZG::setup
 * (g[i] = s^i * G, halo2-base/src/utils/mod.rs:439-443). */
int h2b_g1_fixed_base_mul(h2b_ctx* ctx, const uint64_t base_xy[8], const uint64_t* scalars, size_t n,
                          uint64_t* out_xy);
int h2b_g1_fixed_base_mul_dev(h2b_ctx* ctx, const uint64_t base_xy[8], const void* d_scalars, size_t n,
                              void* d_out_xy);

/* ---- multi-GPU: all-reduce of partial commitments over NVLink peer memory (one process per GPU) ------------------
 * Every rank creates a mailbox and exports its 64-byte CUDA IPC handle; the handles of all ranks (rank order) are
 * exchanged by the caller's process layer (e.g. one torch.distributed all_gather at start-up) and connected once.
 * h2b_g1_allreduce_dev then replaces `all-gather + h2b_g1_sum` by ONE kernel: each rank stores its m partial points
 * (m x 12 limbs, Jacobian) straight into every peer's mailbox through the NVLink-mapped address, publishes a flag,
 * waits for its peers' flags and adds the points; on return (stream order) d_points_xyz holds the m full sums on
 * every rank.  All ranks must call it the same number of times, with the same m.  m <= 16. */
int h2b_peer_create(h2b_ctx* ctx, int rank, int nranks, uint8_t handle_out[64]);
int h2b_peer_connect(h2b_ctx* ctx, const uint8_t* handles /* nranks x 64 bytes */);
int h2b_g1_allreduce_dev(h2b_ctx* ctx, void* d_points_xyz, size_t m);

/* ---- NTT: replaces halo2-axiom 0.5.3 arithmetic::best_fft and poly::EvaluationDomain (SURVEY.md a3) -- */
/* best_fft(a, omega, log_n): in place, natural order in and out, out[i] = sum_j a[j] * omega^(i*j).
 * scale_by_n_inv != 0 additionally multiplies by 2^-log_n (EvaluationDomain::ifft). */
int h2b_ntt_fr(h2b_ctx* ctx, uint64_t* a, uint32_t log_n, const uint64_t omega[4], int scale_by_n_inv);
int h2b_ntt_fr_dev(h2b_ctx* ctx, void* d_a, uint32_t log_n, const uint64_t omega[4], int scale_by_n_inv);
/* omega of the 2^k domain (ROOT_OF_UNITY^(2^(28-k))), Montgomery limbs. */
int h2b_domain_omega(uint32_t k, uint64_t omega_out[4]);
/* EvaluationDomain::lagrange_to_coeff / coeff_to_lagrange on the 2^k domain, in place. */
int h2b_lagrange_to_coeff(h2b_ctx* ctx, uint64_t* a, uint32_t k);
int h2b_coeff_to_lagrange(h2b_ctx* ctx, uint64_t* a, uint32_t k);
int h2b_lagrange_to_coeff_dev(h2b_ctx* ctx, void* d_a, uint32_t k);
int h2b_coeff_to_lagrange_dev(h2b_ctx* ctx, void* d_a, uint32_t k);
/* EvaluationDomain::coeff_to_extended: coeffs[i] *= zeta^(i mod 3), zero-pad n_coeffs -> 2^ext_k,
 * best_fft(extended_omega).  out holds 2^ext_k elements. */
int h2b_coeff_to_extended(h2b_ctx* ctx, const uint64_t* coeffs, size_t n_coeffs, uint32_t ext_k, uint64_t* out);
int h2b_coeff_to_extended_dev(h2b_ctx* ctx, const void* d_coeffs, size_t n_coeffs, uint32_t ext_k, void* d_out);
/* EvaluationDomain::extended_to_coeff: best_fft(extended_omega^-1), scale by 2^-ext_k, a[i] *= zeta^-(i mod 3),
 * in place on 2^ext_k elements (the caller truncates to n*(d-1)). */
int h2b_extended_to_coeff(h2b_ctx* ctx, uint64_t* a, uint32_t ext_k);
int h2b_extended_to_coeff_dev(h2b_ctx* ctx, void* d_a, uint32_t ext_k);

/* Batched forms (halo2 maps these over all columns of a phase): m transforms pipelined through three device
 * buffers so that the PCIe upload of column i+1 and the download of column i-1 overlap the kernels of column i.
 * a[i] / coeffs[i] / out[i] are host pointers (pinned memory makes the copies truly asynchronous). */
int h2b_lagrange_to_coeff_batch(h2b_ctx* ctx, uint64_t* const* a, size_t m, uint32_t k);
int h2b_coeff_to_lagrange_batch(h2b_ctx* ctx, uint64_t* const* a, size_t m, uint32_t k);
/* `domain.lagrange_to_coeff(p)` followed by `domain.coeff_to_extended(p)` for the same m columns (what create_proof does
 * with every advice / permuted / product column): a[j] holds the 2^k Lagrange values on entry and the coefficients on
 * return, ext_out[j] receives the 2^ext_k coset evaluations.  The coefficients cross PCIe once in each direction. */
int h2b_lagrange_to_coeff_and_extended_batch(h2b_ctx* ctx, uint64_t* const* a, size_t m, uint32_t k, uint32_t ext_k,
                                             uint64_t* const* ext_out);
int h2b_coeff_to_extended_batch(h2b_ctx* ctx, const uint64_t* const* coeffs, size_t m, size_t n_coeffs, uint32_t ext_k,
                                uint64_t* const* out);

/* ---- witness assignment: replaces the per-cell loop of assign_witnesses
 *      (halo2-base/src/gates/flex_gate/threads/single_phase.rs:273-312 -> utils/halo2.rs:20-27) ------ */
/* vcol = concatenation of ctx.advice over all threads (N x 4 limbs, `Trivial` payloads); break_points =
 * the pinned ThreadBreakPoints of the phase; cols = ncols x 2^k x 4 limbs, fully written (unassigned rows
 * zero).  H2B_ERR_LAYOUT where the Rust loop panics (break point walks past the last column, or a column
 * overflows 2^k rows, or cells exist with ncols == 0). */
int h2b_assign_columns(h2b_ctx* ctx, const uint64_t* vcol, size_t N, const uint64_t* break_points, size_t nbp,
                       uint32_t k, size_t ncols, uint64_t* cols);
int h2b_assign_columns_dev(h2b_ctx* ctx, const void* d_vcol, size_t N, const uint64_t* break_points,
                           size_t nbp, uint32_t k, size_t ncols, void* d_cols);
/* The same, fed with what halo2-base actually holds: `Vec<Assigned<Fr>>` (halo2-base/src/lib.rs:157-188; enum
 * Zero | Trivial(F) | Rational(F, F)), staged as N records of 72 bytes = 9 x u64: { tag (0 Zero, 1 Trivial, 2 Rational),
 * numerator[4], denominator[4] } (Montgomery limbs; fields a tag does not use are ignored).  The library flattens the
 * cells itself — Rational cells through ONE batched inversion, denominator 0 -> 0 as `batch_invert_assigned` does — and
 * then lays the columns out as h2b_assign_columns.  H2B_ERR_ARG for any other tag (host-pointer form). */
int h2b_assign_columns_assigned(h2b_ctx* ctx, const uint64_t* cells, size_t N, const uint64_t* break_points, size_t nbp,
                                uint32_t k, size_t ncols, uint64_t* cols);
int h2b_assign_columns_assigned_dev(h2b_ctx* ctx, const void* d_cells, size_t N, const uint64_t* break_points,
                                    size_t nbp, uint32_t k, size_t ncols, void* d_cols);
/* LookupAnyManager::assign_raw (halo2-base/src/virtual_region/lookups.rs:130-155): value j -> lookup
 * column j mod L, row j div L.  cols = L x 2^k x 4 limbs. */
int h2b_assign_lookups(h2b_ctx* ctx, const uint64_t* vals, size_t N, uint32_t k, size_t L, uint64_t* cols);
int h2b_assign_lookups_dev(h2b_ctx* ctx, const void* d_vals, size_t N, uint32_t k, size_t L, void* d_cols);
/* Assigned::Rational cells (halo2-base/src/lib.rs:59-60,249-251): out[i] = num[i] * den[i]^-1, den = 0 -> 0
 * (what the prover's batch_invert_assigned yields before committing). */
int h2b_eval_rational(h2b_ctx* ctx, const uint64_t* num, const uint64_t* den, size_t n, uint64_t* out);
int h2b_eval_rational_dev(h2b_ctx* ctx, const void* d_num, const void* d_den, size_t n, void* d_out);
/* The halo2-base form of the witness, as one walk over ctx.advice yields it without inverting anything:
 *   values  N cells: Zero -> 0, Trivial(x) -> x, Rational(n, d) -> n;
 *   index / den  R pairs (uint64 virtual-column index, Montgomery d), one per Rational cell, indices strictly increasing;
 *   lookup index  n_lookup uint64 virtual-column indices in LookupAnyManager::assign_raw order (the cells it copies).
 * h2b_apply_rational_dev turns values into what `batch_invert_assigned` yields: values[index[i]] *= den[i]^-1, d = 0 -> 0.
 * den is overwritten with its inverses.  h2b_assign_lookups_indexed_dev writes values[index[j]] to lookup column j mod L,
 * row j div L, zero elsewhere, as h2b_assign_lookups (same H2B_ERR_LAYOUT rule).  Both are asynchronous: they zero the
 * caller's device verdict word *d_status first and set bit 0 for an index >= N; apply_rational also sets bit 1 for an index
 * not greater than the one before it.  A call with a non-zero verdict leaves its output undefined. */
int h2b_apply_rational_dev(h2b_ctx* ctx, void* d_values, size_t N, const void* d_index, void* d_den, size_t R, uint32_t* d_status);
int h2b_assign_lookups_indexed_dev(h2b_ctx* ctx, const void* d_values, size_t N, const void* d_index, size_t n_lookup, uint32_t k, size_t L,
                                   void* d_cols, uint32_t* d_status);

/* ---- grand-product primitives (SURVEY.md §8(f) rank 2: permutation / lookup arguments of create_proof, §3.3 step 4) */
/* ff 0.13 `BatchInvert::batch_invert`: a[i] <- a[i]^-1 in place, zeros stay zero. */
int h2b_batch_invert_fr(h2b_ctx* ctx, uint64_t* a, size_t n);
int h2b_batch_invert_fr_dev(h2b_ctx* ctx, void* d_a, size_t n);
/* The product column of halo2's permutation / lookup provers: z[0] = start, z[i] = z[i-1] * f[i-1] for i < n
 * (`z.push(z[row - 1] * modified_values[row - 1])`; f[n-1] is not used).  f and z hold n elements. */
int h2b_grand_product_fr(h2b_ctx* ctx, const uint64_t* f, const uint64_t start[4], size_t n, uint64_t* z);
int h2b_grand_product_fr_dev(h2b_ctx* ctx, const void* d_f, const uint64_t start[4], size_t n, void* d_z);

/* The lookup argument's permuted columns: halo2-axiom 0.5.3 plonk/lookup/prover.rs `permute_expression_pair` (not
 * vendored; restated).  input / table: the compressed expressions, 2^k rows (Lagrange form).  Over the usable rows
 * u = 2^k - (blinding_factors + 1): permuted_input = input sorted by Fr's Ord (canonical integer order);
 * permuted_table[row] = permuted_input[row] where a run starts, and the left-over table values (the sorted table minus the
 * first instance of every distinct input value) — ascending — on the repeated rows, front to back (the sorted-table walk
 * of PSE halo2 and its forks, recalled for halo2-axiom 0.5.3) or, with option "lookup.leftover_order" = 1, from the last
 * repeated row backwards (zcash halo2's BTreeMap + pop).  Both satisfy the argument; the choice only shows in the proof
 * bytes.  Rows >= u of both outputs are NOT written (the prover puts its blinding scalars there).  Outputs must not alias inputs.  H2B_ERR_UNSATISFIED when an input value is missing from the table.
 * The `_dev` form synchronises the stream (it has to read the verdict); `_async_dev` does not: it enqueues everything and
 * leaves the verdict in the caller's device word *d_status (0 = satisfied; bit 0 = an input value is missing from the
 * table), to be read whenever the caller next synchronises (the resident prover reads it with the proof's evaluations). */
int h2b_permute_expression_pair(h2b_ctx* ctx, const uint64_t* input, const uint64_t* table, uint32_t k, uint32_t blinding_factors,
                                uint64_t* permuted_input, uint64_t* permuted_table);
int h2b_permute_expression_pair_dev(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, uint32_t blinding_factors,
                                    void* d_permuted_input, void* d_permuted_table);
int h2b_permute_expression_pair_async_dev(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, uint32_t blinding_factors,
                                          void* d_permuted_input, void* d_permuted_table, uint32_t* d_status);

/* ---- quotient evaluation, first slice (SURVEY.md §8(f) rank 1): the custom-gate term of halo2-base's vertical gate
 * `q * (a + b*c - out)` (halo2-base/src/gates/flex_gate/mod.rs:80-91) on the extended coset domain, folded as the
 * prover folds gate terms: acc[i] <- acc[i] * y + q[i] * (a[i] + a[i+s] * a[i+2s] - a[i+3s]), s = 2^(ext_k - k),
 * indices mod 2^ext_k.  q_ext, a_ext, acc: 2^ext_k elements (coeff_to_extended outputs). */
int h2b_flex_gate_fold(h2b_ctx* ctx, const uint64_t* q_ext, const uint64_t* a_ext, const uint64_t y[4], uint32_t k,
                       uint32_t ext_k, uint64_t* acc);
int h2b_flex_gate_fold_dev(h2b_ctx* ctx, const void* d_q_ext, const void* d_a_ext, const uint64_t y[4], uint32_t k,
                           uint32_t ext_k, void* d_acc);

/* ---- quotient evaluation, general form (SURVEY.md §8(f) rank 1): halo2-axiom 0.5.3 `plonk/evaluation.rs`
 * (`Evaluator::evaluate_h`; not vendored — restated from the upstream algorithm, parity unpinned like the rest of L0).
 * All columns are evaluations on the extended coset domain (2^ext_k x [u64;4], outputs of coeff_to_extended); a
 * rotation by r rows of the 2^k domain is the index (i + r * 2^(ext_k-k)) mod 2^ext_k (`get_rotation_idx`).
 *
 * h2b_graph mirrors `GraphEvaluator`: a straight-line program whose calculation number t writes intermediate t.
 *   value source word:  kind | index << 4 | rotation_slot << 20
 *   program:            H2B_CALC_* opcode followed by its value-source words;
 *                       H2B_CALC_HORNER: start, factor, n_parts, parts[n_parts]  ->  ((start*f + p0)*f + p1)...
 * The `_dev` entry points take column tables that are HOST arrays of DEVICE pointers; the host-pointer forms take
 * host columns and stage them (use them for tests / small circuits — the prover keeps these columns resident). */
#define H2B_SRC_CONSTANT 0u
#define H2B_SRC_INTERMEDIATE 1u
#define H2B_SRC_FIXED 2u
#define H2B_SRC_ADVICE 3u
#define H2B_SRC_INSTANCE 4u
#define H2B_SRC_CHALLENGE 5u
#define H2B_SRC_BETA 6u
#define H2B_SRC_GAMMA 7u
#define H2B_SRC_THETA 8u
#define H2B_SRC_Y 9u
#define H2B_SRC_PREVIOUS 10u
#define H2B_SRC(kind, index, rot_slot) ((uint32_t)(kind) | ((uint32_t)(index) << 4) | ((uint32_t)(rot_slot) << 20))
#define H2B_CALC_ADD 0u
#define H2B_CALC_SUB 1u
#define H2B_CALC_MUL 2u
#define H2B_CALC_SQUARE 3u
#define H2B_CALC_DOUBLE 4u
#define H2B_CALC_NEGATE 5u
#define H2B_CALC_HORNER 6u
#define H2B_CALC_STORE 7u
#define H2B_GRAPH_MAX_CALCULATIONS 64
typedef struct h2b_graph {
    const uint32_t* program;     /* host memory */
    size_t program_words;
    uint32_t n_calculations;     /* <= H2B_GRAPH_MAX_CALCULATIONS */
    uint32_t result;             /* value source word of the result */
    const uint64_t* constants;   /* host, n_constants x 4 (Montgomery) */
    size_t n_constants;
    const int32_t* rotations;    /* host, rotation of each rotation slot, in rows of the 2^k domain */
    size_t n_rotations;
    const void* const* fixed;    /* column tables: n_* pointers to 2^ext_k x 4 u64 */
    size_t n_fixed;
    const void* const* advice;
    size_t n_advice;
    const void* const* instance;
    size_t n_instance;
    const uint64_t* challenges;  /* host, n_challenges x 4 */
    size_t n_challenges;
    uint64_t beta[4], gamma[4], theta[4], y[4];
} h2b_graph;
/* custom gates: values[i] <- graph(previous = values[i]) for every row of the extended domain */
int h2b_quotient_graph(h2b_ctx* ctx, const h2b_graph* graph, uint32_t k, uint32_t ext_k, uint64_t* values);
int h2b_quotient_graph_dev(h2b_ctx* ctx, const h2b_graph* graph, uint32_t k, uint32_t ext_k, void* d_values);
/* permutation argument terms of evaluate_h, folded with y in halo2's order:
 *   l_0 (1 - z_0);  l_last (z_last^2 - z_last);  l_0 (z_s - z_{s-1}(omega^last X)) for s >= 1;
 *   l_active (z_s(omega X) prod_j (v_j + beta sigma_j + gamma) - z_s prod_j (v_j + delta^j beta X + gamma)) per set,
 * sets = chunks of `chunk_len` (= degree - 2) permutation columns; last = -(blinding_factors + 1).
 * z: n_sets product cosets; columns / sigma: n_cols value cosets and permutation-polynomial cosets in the
 * permutation's column order.  No-op when n_sets == 0, as in halo2. */
int h2b_permutation_fold(h2b_ctx* ctx, const uint64_t* const* z, size_t n_sets, const uint64_t* const* columns,
                         const uint64_t* const* sigma, size_t n_cols, size_t chunk_len, const uint64_t* l0,
                         const uint64_t* l_last, const uint64_t* l_active, const uint64_t beta[4], const uint64_t gamma[4],
                         const uint64_t y[4], uint32_t blinding_factors, uint32_t k, uint32_t ext_k, uint64_t* values);
int h2b_permutation_fold_dev(h2b_ctx* ctx, const void* const* d_z, size_t n_sets, const void* const* d_columns,
                             const void* const* d_sigma, size_t n_cols, size_t chunk_len, const void* d_l0,
                             const void* d_l_last, const void* d_l_active, const uint64_t beta[4], const uint64_t gamma[4],
                             const uint64_t y[4], uint32_t blinding_factors, uint32_t k, uint32_t ext_k, void* d_values);
/* one lookup argument's five terms; `graph` yields (compressed input + beta)(compressed table + gamma) per row
 * (its beta / gamma / theta / y are the ones used for the fold):
 *   l_0 (1 - z); l_last (z^2 - z); l_active (z(omega X)(a' + beta)(s' + gamma) - z * graph); l_0 (a' - s');
 *   l_active (a' - s')(a' - a'(omega^-1 X)) */
int h2b_lookup_fold(h2b_ctx* ctx, const h2b_graph* graph, const uint64_t* z, const uint64_t* permuted_input,
                    const uint64_t* permuted_table, const uint64_t* l0, const uint64_t* l_last, const uint64_t* l_active,
                    uint32_t k, uint32_t ext_k, uint64_t* values);
int h2b_lookup_fold_dev(h2b_ctx* ctx, const h2b_graph* graph, const void* d_z, const void* d_permuted_input,
                        const void* d_permuted_table, const void* d_l0, const void* d_l_last, const void* d_l_active,
                        uint32_t k, uint32_t ext_k, void* d_values);

/* `EvaluationDomain::divide_by_vanishing_poly`: values[i] *= 1 / t(zeta * extended_omega^i), t(X) = X^(2^k) - 1 — the
 * last pointwise step of the quotient before extended_to_coeff and the split into h pieces.  Requires ext_k > k. */
int h2b_divide_by_vanishing_poly(h2b_ctx* ctx, uint64_t* values, uint32_t k, uint32_t ext_k);
int h2b_divide_by_vanishing_poly_dev(h2b_ctx* ctx, void* d_values, uint32_t k, uint32_t ext_k);

/* ---- constraint check: `MockProver::verify` for halo2-base's constraint system (which gate, lookup or copy constraint a
 * witness breaks, and at which rows) on Lagrange columns of 2^k rows, asynchronous on the context's stream.
 * A report is max_report + 1 uint64 words per checked item, in device memory: the failure count, then the first
 * min(count, max_report) failing rows in ascending order, the remaining words zero.  The same inputs give the same bytes.
 * 1 <= k <= 28 and 1 <= max_report <= H2B_CHECK_MAX_REPORT.  Scratch comes from the context's workspaces.
 *   h2b_check_graph_dev       rows r < `rows` (<= 2^k) where the program's result is not zero; the graph runs on columns of 2^k
 *                             rows with rotations mod 2^k (validated as h2b_quotient_graph_dev validates it; PREVIOUS reads 0).
 *   h2b_check_lookup_dev      rows r < `rows` whose input value is not among table rows [0, rows).
 *   h2b_permutation_decode_dev  n_cols sigma columns (the permutation's column order) -> d_map, n_cols x 2^k uint32:
 *                             map[c][r] = c' << k | r' where sigma_c(r) = delta^c' omega^r', c' < n_cols.  An entry of no such
 *                             form is reported in column c's report (d_reports: n_cols reports) and maps to (c, r) itself.
 *                             Needs k + ceil(log2 n_cols) <= 32 and n_cols <= 65535.
 *   h2b_check_copies_dev      cells (c, r), r < 2^k, whose value differs from the value of cell map[c][r] (a map entry naming a
 *                             column >= n_cols counts as a failure); d_columns: host array of n_cols device pointers in the
 *                             permutation's column order; d_reports: n_cols reports. */
#define H2B_CHECK_MAX_REPORT 65536
int h2b_check_graph_dev(h2b_ctx* ctx, const h2b_graph* g, uint32_t k, size_t rows, size_t max_report, void* d_report);
int h2b_check_lookup_dev(h2b_ctx* ctx, const void* d_input, const void* d_table, uint32_t k, size_t rows, size_t max_report,
                         void* d_report);
int h2b_permutation_decode_dev(h2b_ctx* ctx, const void* const* d_sigma, size_t n_cols, uint32_t k, void* d_map,
                               size_t max_report, void* d_reports /* n_cols reports: malformed entries */);
int h2b_check_copies_dev(h2b_ctx* ctx, const void* const* d_columns, const void* d_map, size_t n_cols, uint32_t k,
                         size_t max_report, void* d_reports /* n_cols reports */);

/* ---- MockProver for a halo2-base builder in its keygen form (no SRS, no sigma, no proving key; see h2b200_mock.hpp).
 * Indices are uint64 positions in the virtual column (ctx.advice concatenated over the threads).  All asynchronous.
 *   h2b_mock_selectors_dev        the selector columns of the gate-advice columns: d_q (ncols x 2^k) gets q_c[r] = 1 where the
 *                                 walk of h2b_assign_columns_dev places virtual cell s_c + r in column c and its selector byte
 *                                 (d_selectors, N bytes) is set, 0 elsewhere; a break cell's selector goes to row 0 of the next
 *                                 column only (the walk enables it after the break).  Same H2B_ERR_LAYOUT rules.
 *   h2b_mock_lookup_selector_dev  q_lookup of one gate column (2^k, zeroed first): q[index[i]] = 1.  *d_status (zeroed first):
 *                                 bit 0 an index >= N, bit 1 an index >= max_rows (an unusable row).
 *   h2b_check_equalities_dev      m pairs (a, b) (2 x uint64 each): the equalities whose cells differ -> one report over the pair
 *                                 indices (form of the constraint check reports).  *d_status (zeroed first): bit 0 for an index
 *                                 >= N (its equality is flagged, nothing is read through it).
 *   h2b_check_constants_dev       m pairs (d_consts[i] Montgomery, d_index[i]): cells differing from their constant; the same report
 *                                 and status rules.
 *   h2b_count_distinct_dev        *d_count (device uint32) = the number of distinct values among m Montgomery elements. */
int h2b_mock_selectors_dev(h2b_ctx* ctx, const void* d_selectors, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k,
                           size_t ncols, void* d_q);
int h2b_mock_lookup_selector_dev(h2b_ctx* ctx, const void* d_index, size_t m, size_t N, size_t max_rows, uint32_t k, void* d_q,
                                 uint32_t* d_status);
int h2b_check_equalities_dev(h2b_ctx* ctx, const void* d_cells, size_t N, const void* d_pairs, size_t m, size_t max_report,
                             void* d_report, uint32_t* d_status);
int h2b_check_constants_dev(h2b_ctx* ctx, const void* d_cells, size_t N, const void* d_consts, const void* d_index, size_t m,
                            size_t max_report, void* d_report, uint32_t* d_status);
int h2b_count_distinct_dev(h2b_ctx* ctx, const void* d_values, size_t m, uint32_t* d_count);

/* ---- keygen of a halo2-base builder: the permutation side of keygen_vk / keygen_pk (see h2b200_keygen.hpp, DESIGN.md §4.8,
 * §4.11).  Cells are u32 ids c 2^k + r, c the permutation column in [c, c1.., c{F-1}, a0.., a{A-1}, l0.., l{L-1}, i0.., i{I-1}]
 * order (F constants columns; the calls without _nf have F = 1).  Synchronous; scratch is allocated and freed per call.
 *   h2b_keygen_copies_dev        the constants column and the copy calls of BaseCircuitBuilder::synthesize in halo2-base's order,
 *                                into d_edges (E = nbp + n_lookup + M + Mc u32 pairs): the break copies (a{j+1}, 0) ~ (a_j,
 *                                bp_j) (break_points: host); the lookup copies raw(index[i]) ~ (l{i mod L}, i / L); the M advice
 *                                equalities (d_pairs: uint64 (a, b)) sorted by (a, b); the Mc constant equalities (d_consts:
 *                                Montgomery, d_const_index: uint64 cells) sorted by (canonical constant, cell) as
 *                                (c, the constant's row) ~ raw(cell), the distinct constants placed at rows 0, 1, .. of d_c (2^k,
 *                                zeroed first) in that order.  raw(p): the cell the gate walk assigns virtual index p (a break
 *                                cell belongs to the column it ends).  d_status (2 words): [0] bit 0 a looked-up index >= N, bit 1
 *                                an equality index >= N (nothing read through it); [1] the number of distinct constants (rows of
 *                                d_c >= 2^k are not written).
 *   h2b_keygen_instance_edges_dev  the copies of BaseCircuitBuilder::assign_instances, which follow the ones above: for each
 *                                instance column m < I in order and each row r < n_index[m] (host array), raw(index_m[r]) ~
 *                                (i_m, r), index_m the next n_index[m] uint64 of d_index (the columns back to back), into d_edges
 *                                (n_index[0] + .. + n_index[I-1] u32 pairs; pass the edges after those of h2b_keygen_copies_dev).
 *                                d_status (I words, zeroed first): word m bit 0 an index >= N at a row r <= usable (halo2-base's
 *                                "instance not assigned" comes before that row's copy), bit 1 a row r >= usable (halo2's copy
 *                                fails with NotEnoughRowsAvailable there); such copies are written as (0, 0), which joins nothing.
 *   h2b_keygen_copies_nf_dev     h2b_keygen_copies_dev with F constants columns (num_fixed, F >= 0): distinct constant d goes to
 *                                constants column d mod F, row d div F (left to right, then top to bottom), its copy is
 *                                ((d mod F) 2^k + d div F) ~ raw(cell), and d_c is an F x 2^k block (column after column, zeroed
 *                                first; null when F = 0).  d_status[1] is the number of distinct constants D; ranks >= F 2^k are
 *                                not written (with F = 0 none is: D > 0 is halo2-base's index-out-of-bounds panic).
 *   h2b_keygen_instance_edges_nf_dev  h2b_keygen_instance_edges_dev with F constants columns before the advice columns.
 *   h2b_keygen_sigma_map_dev     the mapping halo2's permutation Assembly builds from E copies (d_edges, in call order) over
 *                                n_cols x 2^k cells: d_map (n_cols x 2^k u32) = the cell id each cell maps to (as
 *                                h2b_permutation_decode_dev decodes it).  A cell id >= n_cols 2^k is H2B_ERR_ARG.
 *   h2b_keygen_sigma_values_dev  d_sigma (n_cols x 2^k, column after column) = delta^c' omega^r' for d_map's entry c' 2^k + r'. */
int h2b_keygen_copies_dev(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t A, size_t L,
                          const void* d_lookup_index, size_t n_lookup, const void* d_pairs, size_t M, const void* d_consts,
                          const void* d_const_index, size_t Mc, void* d_c, void* d_edges, uint32_t* d_status);
int h2b_keygen_instance_edges_dev(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t A, size_t L,
                                  size_t usable, size_t I, const size_t* n_index, const void* d_index, void* d_edges, uint32_t* d_status);
int h2b_keygen_copies_nf_dev(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t F, size_t A, size_t L,
                             const void* d_lookup_index, size_t n_lookup, const void* d_pairs, size_t M, const void* d_consts,
                             const void* d_const_index, size_t Mc, void* d_c, void* d_edges, uint32_t* d_status);
int h2b_keygen_instance_edges_nf_dev(h2b_ctx* ctx, size_t N, const uint64_t* break_points, size_t nbp, uint32_t k, size_t F, size_t A,
                                     size_t L, size_t usable, size_t I, const size_t* n_index, const void* d_index, void* d_edges,
                                     uint32_t* d_status);
int h2b_keygen_sigma_map_dev(h2b_ctx* ctx, const void* d_edges, size_t E, size_t n_cols, uint32_t k, void* d_map);
int h2b_keygen_sigma_values_dev(h2b_ctx* ctx, const void* d_map, size_t n_cols, uint32_t k, void* d_sigma);

/* ---- selector compression (halo2's keygen_vk with compress_selectors, DESIGN.md §4.13): which selector columns are active on a
 * common row.  S (1 <= S <= H2B_SELECTORS_MAX) selector columns of 2^k Lagrange values each, every value 0 or 1 (Montgomery);
 * conflicts: S x S bytes on the HOST in both forms, row-major, conflicts[i S + j] = 1 iff some row has both i and j set (the
 * diagonal: column i is set on some row), else 0.  A value other than 0 or 1: H2B_ERR_ARG naming the first such column and row
 * (column-major order).  Synchronises. */
#define H2B_SELECTORS_MAX 4096
int h2b_selector_conflicts(h2b_ctx* ctx, const uint64_t* const* selectors, size_t S, uint32_t k, uint8_t* conflicts);
int h2b_selector_conflicts_dev(h2b_ctx* ctx, const void* const* d_selectors, size_t S, uint32_t k, uint8_t* conflicts);

/* ---- opening arithmetic (SURVEY.md §8(f) rank 4): halo2-axiom 0.5.3 `arithmetic::{eval_polynomial, kate_division}`
 * and the polynomial linear combinations of `poly/kzg/multiopen/shplonk/prover.rs` ------------------------------- */
/* out = sum_i coeffs[i] * x^i */
int h2b_eval_polynomial(h2b_ctx* ctx, const uint64_t* coeffs, size_t n, const uint64_t x[4], uint64_t out[4]);
int h2b_eval_polynomial_dev(h2b_ctx* ctx, const void* d_coeffs, size_t n, const uint64_t x[4], uint64_t out[4]);
/* quotient of a(X) (n coefficients, n >= 1) by (X - z): q has n - 1 coefficients, the remainder a(z) is dropped,
 * as `kate_division(a, z)` does. */
int h2b_kate_division(h2b_ctx* ctx, const uint64_t* a, size_t n, const uint64_t z[4], uint64_t* q);
int h2b_kate_division_dev(h2b_ctx* ctx, const void* d_a, size_t n, const uint64_t z[4], void* d_q);
/* quotient of a(X) (n coefficients, n >= 1) by Z_T(X) = prod_j (X - points[j]) for 1 <= m <= H2B_KATE_MULTI_MAX distinct
 * points, the remainder dropped (SHPLONK's div_by_vanishing), in one pass: q = sum_j weights[j] (a - a(z_j)) / (X - z_j) with
 * weights[j] = 1 / prod_{k != j} (z_j - z_k), which the caller supplies (points, weights: m x 4 limbs, host).  q has n - 1
 * coefficients, as kate_division writes them; those from n - m on are zero.  With m = 1 and weight 1 it is kate_division. */
#define H2B_KATE_MULTI_MAX 4
int h2b_kate_division_multi(h2b_ctx* ctx, const uint64_t* a, size_t n, const uint64_t* points, size_t m, const uint64_t* weights,
                            uint64_t* q);
int h2b_kate_division_multi_dev(h2b_ctx* ctx, const void* d_a, size_t n, const uint64_t* points, size_t m, const uint64_t* weights,
                                void* d_q);
/* out[i] = sum_j scalars[j] * polys[j][i], i < n, j < m (1 <= m <= 32); out may alias one of the inputs */
int h2b_poly_lincomb(h2b_ctx* ctx, const uint64_t* const* polys, const uint64_t* scalars, size_t m, size_t n, uint64_t* out);
int h2b_poly_lincomb_dev(h2b_ctx* ctx, const void* const* d_polys, const uint64_t* scalars, size_t m, size_t n, void* d_out);

/* ---- device-resident polynomials (the resident prover path): a column / polynomial of Fr elements that stays in HBM between
 * the calls of one proof — assigned by h2b_assign_columns_dev, committed by h2b_msm_g1_dev, transformed by the `_dev`
 * NTT entry points, consumed by the quotient kernels — so that only commitments, evaluations and blinding scalars cross
 * PCIe.  Replaces the host-side `Polynomial<Fr, _>` vectors of halo2-axiom 0.5.3 plonk/prover.rs (not vendored).
 * h2b_poly_device_ptr() is what every `_dev` entry point takes; offsets / lengths are in elements. */
typedef struct h2b_poly h2b_poly;
int h2b_poly_alloc(h2b_ctx* ctx, size_t n_elems, h2b_poly** out); /* zero-filled */
void h2b_poly_free(h2b_ctx* ctx, h2b_poly* poly);
void* h2b_poly_device_ptr(const h2b_poly* poly);
size_t h2b_poly_len(const h2b_poly* poly);
int h2b_poly_zero(h2b_ctx* ctx, h2b_poly* poly);                                                      /* asynchronous */
/* enqueue only: `pinned_host` must be page-locked and stay untouched until the stream has been synchronised */
int h2b_poly_upload_async(h2b_ctx* ctx, h2b_poly* poly, size_t offset, const uint64_t* pinned_host, size_t n);
int h2b_poly_copy_dev(h2b_ctx* ctx, void* d_dst, const void* d_src, size_t n);                         /* asynchronous, n elements */
int h2b_poly_upload(h2b_ctx* ctx, h2b_poly* poly, size_t offset, const uint64_t* host, size_t n);     /* blocking */
int h2b_poly_download(h2b_ctx* ctx, const h2b_poly* poly, size_t offset, uint64_t* host, size_t n);   /* blocking */

/* ---- product columns of the permutation and lookup arguments (create_proof step 4, SURVEY.md §3.3), built on the device:
 * row factors -> one batched inversion -> prefix products.  u = 2^k - (blinding_factors + 1) usable rows; z[0] = start,
 * z[i + 1] = z[i] * f_i for i < u, z[i] = z[u] above (the caller overwrites rows > u with its blinding scalars).
 * permutation set of n_cols <= 8 columns whose first column has index `first_col` in the permutation's column order:
 *   f_i = prod_j (v_j(i) + beta delta^(first_col + j) omega^i + gamma) / prod_j (v_j(i) + beta sigma_j(i) + gamma);
 *   d_start = NULL for the first set, else a device pointer to the previous set's z[u] (halo2 chains the sets).
 * lookup: f_i = (input_i + beta)(table_i + gamma) / ((permuted_input_i + beta)(permuted_table_i + gamma)). */
int h2b_permutation_product_dev(h2b_ctx* ctx, const void* const* d_columns, const void* const* d_sigma, size_t n_cols,
                                size_t first_col, const uint64_t beta[4], const uint64_t gamma[4], uint32_t k,
                                uint32_t blinding_factors, const void* d_start, void* d_z);
int h2b_lookup_product_dev(h2b_ctx* ctx, const void* d_input, const void* d_table, const void* d_permuted_input,
                           const void* d_permuted_table, const uint64_t beta[4], const uint64_t gamma[4], uint32_t k,
                           uint32_t blinding_factors, void* d_z);
/* out[i] = a[i] * b[i] (out may alias a): compressed lookup input q * a of halo2-base/src/gates/range/mod.rs:131-140 */
int h2b_fr_mul_elementwise_dev(h2b_ctx* ctx, const void* d_a, const void* d_b, size_t n, void* d_out);
/* out[j] = polys[j](xs[j]) for m device polynomials of n coefficients; xs, out: host, m x 4 limbs (one synchronisation) */
int h2b_eval_polynomial_batch_dev(h2b_ctx* ctx, const void* const* d_polys, const uint64_t* xs, size_t m, size_t n,
                                  uint64_t* out);

/* ---- test hooks (field arithmetic of the kernels, element-wise on the device) --------------------- */
/* field: 0 = Fq, 1 = Fr; op: 0 mul, 1 add, 2 sub, 3 inv(a), 4 from_mont(a), 5 to_mont(a), 6 sqr(a),
 * 7 a*b + (a+b)(a-b) and 8 a*b - b*b through the fused two-product Montgomery routine of the group law,
 * 9 inv(a) by the binary extended Euclidean routine the single-lane inversions use,
 * 10 a[i]*b[i] + a[n+i]*b[n+i] through the fused two-product routine with four independent operands (a and b then hold
 * 2n elements each, out n) */
int h2b_test_field_op(h2b_ctx* ctx, int field, int op, const uint64_t* a, const uint64_t* b, size_t n, uint64_t* out);

#ifdef __cplusplus
}
#endif
#endif /* H2B200_H */
