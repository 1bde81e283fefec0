/*
 * spectre_b200.h -- C ABI of libspectre_b200.so, the H100-native backend for the Halo2/KZG create_proof
 * hot path of ChainSafe/Spectre (MSM over BN254 G1, NTT over Fr, EvaluationDomain and batch polynomial ops).
 *
 * This is the drop-in boundary of SURVEY.md section 8b: exactly what a Rust `extern "C"` block in a
 * `[patch]`-ed halo2_proofs would bind (INTEGRATION.md shows that block). Spectre itself reaches these
 * routines only through snark_verifier_sdk::{gen_pk, gen_proof_shplonk, gen_snark_shplonk,
 * gen_evm_proof_shplonk} at lightclient-circuits/src/util/circuit.rs:131,158,177,211,263; the functions
 * replaced live in the un-vendored crate halo2_proofs ([UPSTREAM], reference Cargo.toml:44-48).
 *
 * Data conventions (identical to halo2curves' in-memory types, so `&[Fr]` / `&[G1Affine]` pass as pointers):
 *   spb_fr / spb_fq : 4 x u64 little-endian limbs of a*2^256 mod m (Montgomery form), 32 bytes
 *   spb_g1_affine   : {x, y}, 64 bytes, identity encoded as x = y = 0
 *   spb_g1          : Jacobian {x, y, z}, 96 bytes, affine = (x/z^2, y/z^3), identity z = 0
 * Pointers are HOST pointers unless a function name ends in `_dev`; the library never keeps a caller pointer
 * after returning and never frees caller memory. All functions are thread-safe (one lock per context).
 *
 * Stream contract of the `_dev` entry points: the library enqueues its work on the context's own non-blocking stream
 * of that device (spb_stream) -- MSMs on lane streams that first wait for it -- and returns only after that work has
 * completed, so results are visible to any stream on return. Inputs are the caller's side of the contract: a device
 * buffer passed to a `_dev` call must either have been produced on spb_stream(ctx, i) (enqueue your memsets / copies /
 * kernels there, as include/spectre_b200_prover.hpp's CudaMemory and the Python DeviceEngine do: no synchronisation is
 * needed then) or be complete, i.e. the producing stream synchronised, before the call. The legacy default stream does
 * NOT order against spb_stream (it is created with cudaStreamNonBlocking).
 * Concurrency (Spectre's RPC `--concurrency N`, prover/src/prover.rs:114): one context serialises its calls; open one
 * context per concurrent proof on the same device(s) -- they share nothing but the GPU; every context holds its own handles
 * (tests/test_gpu_msm.py::test_two_contexts_prove_concurrently_on_one_device; one spb_srs used from two contexts is not exercised).
 * Return value: 0 = ok, negative = error (spb_last_error gives the text); nothing aborts or throws.
 * There is no CPU fallback inside the library: without a usable CUDA device spb_init fails.
 */
#ifndef SPECTRE_B200_H
#define SPECTRE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

typedef struct { uint64_t l[4]; } spb_fr;
typedef struct { uint64_t l[4]; } spb_fq;
typedef struct { spb_fq x, y; } spb_g1_affine;
typedef struct { spb_fq x, y, z; } spb_g1;

typedef struct spb_ctx spb_ctx;
typedef struct spb_srs spb_srs;       /* device-resident ParamsKZG: g and g_lagrange */
typedef struct spb_domain spb_domain; /* EvaluationDomain<Fr> constants */

#define SPB_OK 0
#define SPB_ERR_CUDA (-1)
#define SPB_ERR_ARG (-2)
#define SPB_ERR_OOM (-3)
#define SPB_ERR_STATE (-4)
#define SPB_ERR_CONSTRAINT (-5) /* halo2's Error::ConstraintSystemFailure (lookup input not in table) */
#define SPB_ERR_DATA (-6)       /* invalid input data: halo2's io::ErrorKind::InvalidData */

#define SPB_BASIS_G 0          /* monomial basis  (Params::commit)          */
#define SPB_BASIS_G_LAGRANGE 1 /* Lagrange basis  (Params::commit_lagrange) */

/* ---- context -------------------------------------------------------------------------------------------- */
/* One context drives n_dev devices of this process (device_ids == NULL: devices 0..n_dev-1). With n_dev > 1
 * an MSM is sharded by point range over the devices and the partial sums are folded on the host; host-buffer NTTs of
 * 2^16 points and more run six-step across all devices (one NVLink all-to-all), `_dev` NTTs on the first device. Multi-process use (one context per rank, torch.distributed / NCCL between ranks) is
 * what bench.py does. An id may repeat: each entry is a shard with its own stream, workspaces, MSM lanes, twiddle tables and
 * SRS range, and the entries that name the same device share its memory and SMs (one device, several shards). Such a
 * context runs every multi-device path on one GPU and computes the same results; it is how the test suite checks those
 * paths where only one GPU is present. Returns NULL on failure (no CUDA device, bad id). */
spb_ctx* spb_init(const int* device_ids, int n_dev);
void spb_shutdown(spb_ctx* ctx);
/* Free the context's cached device memory -- the grow-only workspaces of MSM, NTT and the provers, and the cached twiddle
 * tables -- after the work queued on its devices is done; later calls allocate again as needed. For a long-lived context
 * that ran large transforms before a proof that needs the memory. Fails while an spb_shplonk handle is open. */
int spb_release_workspace(spb_ctx* ctx);
const char* spb_last_error(spb_ctx* ctx);
/* kernels launched by this context so far, and device milliseconds of the last timed call (CUDA events on the
 * context's own stream, taken inside every spb_msm* / spb_ntt* call). */
uint64_t spb_kernel_launches(spb_ctx* ctx);
float spb_last_device_ms(spb_ctx* ctx);
int spb_device_count(void);
/* The CUDA stream (a cudaStream_t) every `_dev` call of device `dev_index` of this context is ordered on; NULL on a bad
 * index. See "Stream contract" above. */
void* spb_stream(spb_ctx* ctx, int dev_index);
/* File <-> device streaming for the prover's large artefacts (params/kzg_bn254_{k}.srs, *.pkey; reference: .gitignore:34-43,
 * lightclient-circuits/src/util/circuit.rs:104-115,273-280): `bytes` bytes at `offset` of the file go straight to / come from
 * a device buffer of the first device through two pinned staging buffers, the file read of one chunk overlapping the DMA of
 * the previous one. spb_write_file_dev truncates the file unless `append`. */
int spb_read_file_dev(spb_ctx* ctx, const char* path, uint64_t offset, void* d_dst, size_t bytes);
int spb_write_file_dev(spb_ctx* ctx, const char* path, int append, const void* d_src, size_t bytes);
/* pin / unpin a caller buffer so host<->device copies run at full PCIe rate (optional) */
int spb_host_register(spb_ctx* ctx, void* ptr, size_t bytes);
int spb_host_unregister(spb_ctx* ctx, void* ptr);

/* ---- ParamsKZG ------------------------------------------------------------------------------------------- */
/* Replaces holding ParamsKZG<Bn256>{g, g_lagrange} on the host ([UPSTREAM] halo2_proofs/src/poly/kzg/commitment.rs;
 * created by the reference through gen_srs at prover/src/cli.rs:48,64,87,113,141,165,191,218 and
 * prover/src/prover.rs:55). Copies both bases (2^k points each) to the device(s) once; either may be NULL. */
int spb_srs_upload(spb_ctx* ctx, uint32_t k, const spb_g1_affine* g, const spb_g1_affine* g_lagrange, spb_srs** out);
/* ParamsKZG::setup(k, rng) with the secret drawn by the caller: g[i] = s^i G1, g_lagrange[i] = L_i(s) G1,
 * computed on the device (fixed-base scalar multiplication) -- what halo2-base's gen_srs(k) produces when
 * `s` is the first Fr::random of ChaCha20Rng::from_seed([0;32]). */
int spb_srs_setup(spb_ctx* ctx, uint32_t k, const spb_fr* s, spb_srs** out);
/* copy a range of a resident basis back to the host (ParamsKZG::get_g / write) */
int spb_srs_download(spb_ctx* ctx, const spb_srs* srs, int basis, size_t start, size_t count, spb_g1_affine* out);
void spb_srs_free(spb_ctx* ctx, spb_srs* srs);
/* ParamsKZG::downsize(k), k <= the handle's k: g truncated to 2^k points and g_lagrange recomputed for the smaller domain
 * (g_to_lagrange: the inverse DFT over the group, on the device; no knowledge of the secret needed). The reference keeps
 * a degree -> params map for exactly this (prover/src/prover.rs:34). Returns a NEW handle without window tables. */
int spb_srs_downsize(spb_ctx* ctx, const spb_srs* srs, uint32_t k, spb_srs** out);
/* A powers-of-tau update of a 2^k SRS by the secret t (Montgomery limbs, 0 < t < r): a NEW handle (no window tables) with
 * g'[j] = t^j g[j], g_lagrange' = g_to_lagrange(g'), g2' = g2, s_g2' = t s_g2 -- ParamsKZG::setup run by several parties, each
 * of which applies its own t; nobody learns the final secret unless every party's t is known. The input handle is not
 * modified. SPB_ERR_ARG: a NULL argument, t = 0 or t >= r; SPB_ERR_STATE: a spb_bases_upload handle, a handle with window
 * tables, or a handle whose G2 trailer is zero (spb_srs_set_g2 first). spb_last_device_ms: the scaling and g_to_lagrange. */
int spb_srs_contribute(spb_ctx* ctx, const spb_srs* srs, const spb_fr* t, spb_srs** out);
/* ParamsKZG::read_custom / ::write: k (u32 LE) | g[2^k] | g_lagrange[2^k] | g2 | s_g2 with every coordinate as its
 * in-memory Montgomery limbs -- the `params/kzg_bn254_{k}.srs` file halo2-base's gen_srs caches (reference:
 * prover/src/cli.rs:48, .gitignore:36). The read streams the points straight into device memory.
 *   SPB_SERDE_RAW_BYTES: the checked format (upstream's ParamsKZG::read). Every coordinate's stored limbs must be less than
 *     p and every point must lie on its curve (G1: y^2 = x^3 + 3; G2: y^2 = x^3 + 3/(9+u)) or be the identity (0, 0). The
 *     G1 points are checked on the device that holds them, the G2 trailer on the host. Otherwise the call returns
 *     SPB_ERR_DATA and the error text names the first invalid point in file order (g, g_lagrange, g2, s_g2) and the
 *     reason, e.g. "g_lagrange[262144]: not on the curve". spb_last_device_ms then gives the check kernels' device time.
 *   SPB_SERDE_RAW_BYTES_UNCHECKED: no checks.
 * Any other format is SPB_ERR_ARG (the compressed SerdeFormat::Processed is not implemented). On failure *out is untouched. */
#define SPB_SERDE_RAW_BYTES 1
#define SPB_SERDE_RAW_BYTES_UNCHECKED 2
int spb_srs_read_file_custom(spb_ctx* ctx, const char* path, int format, spb_srs** out);
/* spb_srs_read_file_custom(.., SPB_SERDE_RAW_BYTES_UNCHECKED, ..): does NOT validate the points */
int spb_srs_read_file(spb_ctx* ctx, const char* path, spb_srs** out);
int spb_srs_write_file(spb_ctx* ctx, const spb_srs* srs, const char* path);
int spb_srs_set_g2(spb_ctx* ctx, spb_srs* srs, const unsigned char g2[128], const unsigned char s_g2[128]);
int spb_srs_get_g2(spb_ctx* ctx, const spb_srs* srs, unsigned char g2[128], unsigned char s_g2[128]);
uint32_t spb_srs_k(const spb_srs* srs);

/* ---- MSM -------------------------------------------------------------------------------------------------- */
/* best_multiexp(coeffs, bases) -> G1 ([UPSTREAM] halo2_proofs/src/arithmetic.rs): sum_i scalars[i] * bases[i].
 * `out` is the Jacobian point normalised to z = 1 (identity: x = 0, y = 1, z = 0). */
int spb_msm_raw(spb_ctx* ctx, const spb_fr* scalars, const spb_g1_affine* bases, size_t n, spb_g1* out);
/* best_multiexp against bases the caller reuses: upload ANY n bases once (the handle is an SRS handle with only basis SPB_BASIS_G
 * resident; free it with spb_srs_free, widen its window with spb_srs_precompute), then spb_msm / spb_msm_batch(handle, SPB_BASIS_G,
 * ...) move only the 32 B x n of scalars per call instead of spb_msm_raw's 96 B x n. */
int spb_bases_upload(spb_ctx* ctx, const spb_g1_affine* bases, size_t n, spb_srs** out);
/* Params::commit / commit_lagrange: MSM of `n` scalars against the first n points of a resident basis. */
int spb_msm(spb_ctx* ctx, const spb_srs* srs, int basis, const spb_fr* scalars, size_t n, spb_g1* out);
/* same with the scalars already resident on device 0 of the context */
int spb_msm_dev(spb_ctx* ctx, const spb_srs* srs, int basis, const spb_fr* d_scalars, size_t n, spb_g1* out);
/* `count` MSMs of n scalars each against the same resident basis (create_proof commits its advice / permutation /
 * lookup columns back to back against g_lagrange). Consecutive MSMs cycle over three stream lanes so the
 * latency-bound tail of one and the sort of the next overlap the accumulation of the one in between; out[i] belongs to
 * scalars[i]. */
int spb_msm_batch(spb_ctx* ctx, const spb_srs* srs, int basis, const spb_fr* const* scalars, size_t n, size_t count, spb_g1* out);
int spb_msm_batch_dev(spb_ctx* ctx, const spb_srs* srs, int basis, const spb_fr* const* d_scalars, size_t n, size_t count, spb_g1* out);
/* Precompute the 2^(c*j) multiples of the resident bases (W x the basis memory, one-time). Afterwards every MSM on
 * this SRS folds all windows into one bucket set with a wider window (fewer mixed additions, no window Horner).
 * Results are identical; only the schedule changes. Tables that would take more than a quarter of a device's memory are
 * not built (the call succeeds and the SRS keeps one bucket set per window). */
int spb_srs_precompute(spb_ctx* ctx, spb_srs* srs);
/* number of G1 additions (mixed + full) the last MSM executed on the device(s) */
uint64_t spb_last_msm_adds(spb_ctx* ctx);
/* device milliseconds of the last MSM's stages on the context's first device, from CUDA events on the stream the
 * kernels ran on: [0] signed digits into an unsorted entry list, [1] the entry count's trip to the host and the radix sort
 * of the entries by bucket, [2] bucket offsets of the sorted list, [3] bucket accumulation (the dominant kernel), [4] chain stitch, [5] bucket groups (running sums over 8 buckets per thread), [6] row/column tree sums of the
 * group sums + weighted partial sums. */
void spb_last_msm_stage_ms(spb_ctx* ctx, float out[7]);
/* window width c and window count the library uses for an n-pair MSM (tables: with spb_srs_precompute) */
void spb_msm_geometry(size_t n, int tables, uint32_t* c, uint32_t* windows);

/* Sum of n Jacobian points on the host (folding the per-rank / per-device partial results of a sharded MSM after
 * the all-gather; EC addition is not an NCCL reduction). Result normalised to z = 1. No context needed. */
int spb_g1_sum(const spb_g1* pts, size_t n, spb_g1* out);
/* the same for a batch: pts is [groups][count] (one row per rank, as an all-gather delivers it), out[i] = sum over the groups */
int spb_g1_sum_batch(const spb_g1* pts, size_t groups, size_t count, spb_g1* out);

/* ---- NTT -------------------------------------------------------------------------------------------------- */
/* best_fft(a, omega, log_n) ([UPSTREAM] halo2_proofs/src/arithmetic.rs): in place, natural order,
 * a[i] <- sum_j a[j] omega^(ij), no scaling. */
int spb_ntt(spb_ctx* ctx, spb_fr* a, uint32_t log_n, const spb_fr* omega);
int spb_ntt_dev(spb_ctx* ctx, spb_fr* d_a, uint32_t log_n, const spb_fr* omega);

/* ---- EvaluationDomain ([UPSTREAM] halo2_proofs/src/poly/domain.rs) -------------------------------------- */
/* EvaluationDomain::new(j, k) */
int spb_domain_new(spb_ctx* ctx, uint32_t j, uint32_t k, spb_domain** out);
void spb_domain_free(spb_ctx* ctx, spb_domain* d);
uint32_t spb_domain_extended_k(const spb_domain* d);
/* omega, omega_inv, extended_omega, extended_omega_inv, g_coset, g_coset_inv, ifft_divisor, extended_ifft_divisor */
void spb_domain_constants(const spb_domain* d, spb_fr out[8]);
/* lagrange_to_coeff: a (2^k values) in place */
int spb_lagrange_to_coeff(spb_ctx* ctx, const spb_domain* d, spb_fr* a);
/* coeff_to_lagrange: a (2^k values) in place (plain forward transform) */
int spb_coeff_to_lagrange(spb_ctx* ctx, const spb_domain* d, spb_fr* a);
/* coeff_to_extended: in = 2^k coefficients, out = 2^extended_k evaluations on the zeta-coset */
int spb_coeff_to_extended(spb_ctx* ctx, const spb_domain* d, const spb_fr* in, spb_fr* out);
/* extended_to_coeff: in = 2^extended_k evaluations, out = 2^k * (j-1) coefficients */
int spb_extended_to_coeff(spb_ctx* ctx, const spb_domain* d, const spb_fr* in, spb_fr* out);
/* divide_by_vanishing_poly: a (2^extended_k) in place, a[i] *= t_evaluations[i mod 2^(extended_k-k)] */
int spb_divide_by_vanishing(spb_ctx* ctx, const spb_domain* d, spb_fr* a);
/* device-resident variants (pointers on device 0 of the context) */
int spb_lagrange_to_coeff_dev(spb_ctx* ctx, const spb_domain* d, spb_fr* d_a);
int spb_coeff_to_extended_dev(spb_ctx* ctx, const spb_domain* d, const spb_fr* d_in, spb_fr* d_out);
int spb_extended_to_coeff_dev(spb_ctx* ctx, const spb_domain* d, const spb_fr* d_in, spb_fr* d_out);
int spb_divide_by_vanishing_dev(spb_ctx* ctx, const spb_domain* d, spb_fr* d_a);
/* `count` polynomials at once (create_proof converts its advice / permutation / lookup columns back to back): on a
 * context with several devices polynomial i runs on device i mod n_dev, reading and writing the caller's buffers on the
 * first device through NVLink peer access (SURVEY.md 8e: NTTs sharded by polynomial). HOST arrays of device pointers. */
int spb_lagrange_to_coeff_batch_dev(spb_ctx* ctx, const spb_domain* d, spb_fr* const* d_a, size_t count);
int spb_coeff_to_extended_batch_dev(spb_ctx* ctx, const spb_domain* d, const spb_fr* const* d_in, spb_fr* const* d_out, size_t count);
/* Coset part `part` of coeff_to_extended, for evaluating the quotient one n-row part at a time. With R = 2^(extended_k - k),
 * d_out[i][m] = coeff_to_extended(d_in[i])[part + R m] for m < 2^k: the values at g omega^m, g = zeta extended_omega^part,
 * computed as one 2^k-point transform of the coefficients pre-scaled by g^a. Out of place (d_in is never written); spread over
 * the devices like spb_coeff_to_extended_batch_dev. part >= R: SPB_ERR_ARG. HOST arrays of device pointers. */
int spb_coeff_to_extended_part_batch_dev(spb_ctx* ctx, const spb_domain* d, uint32_t part, const spb_fr* const* d_in, spb_fr* const* d_out, size_t count);
/* d_extended[part + R m] = d_part[m] for m < 2^k: a coset part back into its rows of a 2^extended_k buffer. Rows are sharded
 * over the context's devices like the quotient passes. part >= R: SPB_ERR_ARG. */
int spb_extended_part_scatter_dev(spb_ctx* ctx, const spb_domain* d, uint32_t part, const spb_fr* d_part, spb_fr* d_extended);

/* ---- batch polynomial arithmetic ([UPSTREAM] halo2_proofs/src/arithmetic.rs, ff::BatchInvert) ---------- */
/* Zero-length inputs: with n = 0, spb_vec_{mul,axpy,scale}, spb_grand_product, spb_batch_invert (host and _dev forms),
 * spb_grand_product_seeded_dev, spb_fr_random_chacha_dev, spb_lincomb_dev, spb_weighted_sum_dev and spb_g1_fixed_base_mul
 * return 0 without touching the device; spb_eval_polynomial(_dev) returns 0 with *out = 0. */
/* a[i] <- a[i]^-1, zeros stay zero (BatchInvert semantics) */
int spb_batch_invert(spb_ctx* ctx, spb_fr* a, size_t n);
/* eval_polynomial(poly, point) */
int spb_eval_polynomial(spb_ctx* ctx, const spb_fr* poly, size_t n, const spb_fr* point, spb_fr* out);
/* kate_division(a, b): q (n-1 values) = a(X) / (X - b), remainder dropped */
int spb_kate_division(spb_ctx* ctx, const spb_fr* a, size_t n, const spb_fr* b, spb_fr* q);
/* running product z[0] = 1, z[i+1] = z[i] * a[i]  (the permutation / lookup grand-product scan), n values in, n out */
int spb_grand_product(spb_ctx* ctx, const spb_fr* a, size_t n, spb_fr* z);
/* out[i] = a[i] * b[i] + c * d[i]  style helpers are built by the caller from: */
int spb_vec_mul(spb_ctx* ctx, spb_fr* a, const spb_fr* b, size_t n);                 /* a[i] *= b[i]        */
int spb_vec_axpy(spb_ctx* ctx, spb_fr* y, const spb_fr* alpha, const spb_fr* x, size_t n); /* y[i] += alpha*x[i] */
int spb_vec_scale(spb_ctx* ctx, spb_fr* a, const spb_fr* alpha, size_t n);           /* a[i] *= alpha       */

/* device-resident variants of the batch ops (pointers on device 0 of the context; scalars / results on the host) */
int spb_batch_invert_dev(spb_ctx* ctx, spb_fr* d_a, size_t n);
int spb_eval_polynomial_dev(spb_ctx* ctx, const spb_fr* d_poly, size_t n, const spb_fr* point, spb_fr* out);
/* out[q] = d_polys[q](points[q]) for `count` queries of n coefficients each in one launch (create_proof's evaluation stage
 * after squeezing x: every opened polynomial at every queried rotation). d_polys: HOST array of device pointers. */
int spb_eval_polynomial_many_dev(spb_ctx* ctx, const spb_fr* const* d_polys, size_t n, const spb_fr* points, size_t count, spb_fr* out);
/* d_out[i] = the (first + i)-th draw of `Fr::random(&mut ChaCha20Rng::from_seed(seed))` ([UPSTREAM] rand_chacha + halo2curves
 * Fr::random = from_u512 of one 64-byte keystream block), generated on the device: the vanishing argument's random polynomial
 * (2^k coefficients; [UPSTREAM] plonk/vanishing/prover.rs `commit`) and any other bulk randomness of create_proof need not be
 * drawn on the host or cross PCIe. The same seed on a CPU ChaCha20Rng yields the same elements. */
int spb_fr_random_chacha_dev(spb_ctx* ctx, const uint8_t seed[32], uint64_t first, spb_fr* d_out, size_t n);
int spb_kate_division_dev(spb_ctx* ctx, const spb_fr* d_a, size_t n, const spb_fr* b, spb_fr* d_q);
int spb_grand_product_dev(spb_ctx* ctx, const spb_fr* d_a, size_t n, spb_fr* d_z);
/* row-sharded grand product (SURVEY.md 8e): each rank takes spb_product_dev of its rows, the 32-byte totals are
 * exchanged, and the rank scans its rows seeded with the product of the totals before it:
 * d_z[i] = init * prod_{j<i} d_a[j]. */
int spb_product_dev(spb_ctx* ctx, const spb_fr* d_a, size_t n, spb_fr* out);
int spb_grand_product_seeded_dev(spb_ctx* ctx, const spb_fr* d_a, size_t n, const spb_fr* init, spb_fr* d_z);
int spb_vec_mul_dev(spb_ctx* ctx, spb_fr* d_a, const spb_fr* d_b, size_t n);
int spb_vec_axpy_dev(spb_ctx* ctx, spb_fr* d_y, const spb_fr* alpha, const spb_fr* d_x, size_t n);
int spb_vec_scale_dev(spb_ctx* ctx, spb_fr* d_a, const spb_fr* alpha, size_t n);
/* d_out[i] = sum_p y^p * d_polys[p][i]: the fold-with-powers-of-y that evaluate_h, vanishing::evaluate and the
 * SHPLONK opener apply to sets of polynomials. d_polys is a HOST array of `count` device pointers; d_out may alias
 * none of them. One streaming pass over every input. */
int spb_lincomb_dev(spb_ctx* ctx, const spb_fr* const* d_polys, size_t count, const spb_fr* y, spb_fr* d_out, size_t n);

/* ---- quotient numerator ([UPSTREAM] halo2_proofs/src/plonk/evaluation.rs: GraphEvaluator, Evaluator::evaluate_h) ---- */
/* The gate graph in the flat encoding the Rust shim emits from GraphEvaluator's `calculations`:
 *   per calculation: word0 = op | nparts << 8  (op: 0 Add 1 Sub 2 Mul 3 Square 4 Double 5 Negate 6 Horner 7 Store),
 *                    word1 = target intermediate, then sources of two words each: kind, idx | rot_idx << 16
 *   kind: 0 Constant 1 Intermediate 2 Fixed 3 Advice 4 Instance 5 Challenge 6 Beta 7 Gamma 8 Theta 9 Y 10 PreviousValue
 *   Add/Sub/Mul: a, b.  Square/Double/Negate/Store: a.  Horner: start, factor, then nparts parts. */
typedef struct {
  const uint32_t* program;
  size_t program_words;
  uint32_t num_calculations, num_intermediates;
  const spb_fr* constants;
  uint32_t num_constants;
  const int32_t* rotations;
  uint32_t num_rotations;
} spb_graph;
/* values[idx] <- graph(idx) for every extended row idx < size (PreviousValue = the old values[idx]); column arrays are
 * HOST arrays of device pointers to extended-coset polynomials; rot_scale = 2^(extended_k - k). */
int spb_graph_evaluate_dev(spb_ctx* ctx, const spb_graph* g, const spb_fr* const* d_fixed, uint32_t n_fixed, const spb_fr* const* d_advice, uint32_t n_advice,
                           const spb_fr* const* d_instance, uint32_t n_instance, const spb_fr* challenges, uint32_t n_challenges, const spb_fr* beta,
                           const spb_fr* gamma, const spb_fr* theta, const spb_fr* y, spb_fr* d_values, uint64_t size, int32_t rot_scale);
/* permutation-argument terms of evaluate_h folded into values with powers of y. d_z: n_sets product cosets; d_col_values /
 * d_sigma: the n_cols permuted columns' value and sigma cosets in permutation order (chunk_len per set). */
int spb_permutation_constraints_dev(spb_ctx* ctx, spb_fr* d_values, uint64_t size, int32_t rot_scale, int32_t last_rotation, uint32_t n_sets, uint32_t chunk_len,
                                    const spb_fr* const* d_z, uint32_t n_cols, const spb_fr* const* d_col_values, const spb_fr* const* d_sigma,
                                    const spb_fr* d_l0, const spb_fr* d_l_last, const spb_fr* d_l_active, const spb_fr* beta, const spb_fr* gamma,
                                    const spb_fr* y, const spb_fr* extended_omega);
/* the same terms with X = coset_generator * omega^idx at row idx: over coset part j of the extended coset (size = 2^k,
 * rot_scale = 1, every input a part from spb_coeff_to_extended_part_batch_dev) coset_generator = zeta extended_omega^j and
 * omega = the 2^k-th root. (zeta, extended_omega) gives spb_permutation_constraints_dev. */
int spb_permutation_constraints_coset_dev(spb_ctx* ctx, spb_fr* d_values, uint64_t size, int32_t rot_scale, int32_t last_rotation, uint32_t n_sets,
                                          uint32_t chunk_len, const spb_fr* const* d_z, uint32_t n_cols, const spb_fr* const* d_col_values,
                                          const spb_fr* const* d_sigma, const spb_fr* d_l0, const spb_fr* d_l_last, const spb_fr* d_l_active,
                                          const spb_fr* beta, const spb_fr* gamma, const spb_fr* y, const spb_fr* coset_generator, const spb_fr* omega);
/* the five lookup-argument terms of one lookup; d_table_value[idx] = (compressed input + beta)(compressed table + gamma) */
int spb_lookup_constraints_dev(spb_ctx* ctx, spb_fr* d_values, uint64_t size, int32_t rot_scale, const spb_fr* d_product, const spb_fr* d_permuted_input,
                               const spb_fr* d_permuted_table, const spb_fr* d_table_value, const spb_fr* d_l0, const spb_fr* d_l_last,
                               const spb_fr* d_l_active, const spb_fr* beta, const spb_fr* gamma, const spb_fr* y);

/* ---- lookup argument ([UPSTREAM] halo2_proofs/src/plonk/lookup/prover.rs) ------------------------------------------ */
/* permute_expression_pair over the `usable` rows (blinding rows are appended by the caller from its RNG):
 * d_permuted_input = input values sorted by canonical integer; d_permuted_table = the table values rearranged so that
 * every row satisfies a' == s' or a' == a'[row-1], exactly as the CPU algorithm arranges them.
 * Returns SPB_ERR_CONSTRAINT when an input value does not occur in the table. */
int spb_permute_expression_pair_dev(spb_ctx* ctx, const spb_fr* d_input, const spb_fr* d_table, size_t usable, spb_fr* d_permuted_input, spb_fr* d_permuted_table);

/* ---- witness check ([UPSTREAM] halo2_proofs/src/dev.rs, MockProver::verify) ------------------------------------------ */
/* Each of the three reports the first `cap` failing rows in ascending order and the exact count of failing rows; only those
 * cross PCIe. Inputs are device buffers of the context's first device and are not written; outputs are HOST arrays, filled
 * before the call returns. A NULL context, or a NULL pointer the call would read or write, is SPB_ERR_ARG. A call with no
 * rows to check launches nothing and reports 0.
 * Kernel launches (spb_kernel_launches): spb_nonzero_rows_dev 2; spb_lookup_missing_rows_dev 12 + 2 per non-trivial digit
 * pass of the table's radix sort (a pass runs for each byte of each 64-bit limb of the canonical values on which the usable
 * table rows do not all agree); spb_copy_mismatches_dev 2 per column. */
/* rows_out[0 .. min(cap, total)) = the rows r in [lo, hi) with d_values[r] != 0, ascending; *total_out = their number.
 * hi must be below 2^32. Used on a gate evaluated over the n Lagrange rows. */
int spb_nonzero_rows_dev(spb_ctx* ctx, const spb_fr* d_values, uint64_t lo, uint64_t hi, uint32_t cap, uint32_t* rows_out, uint64_t* total_out);
/* Lookup membership: the rows r < usable whose d_input[r] equals no d_table[j], j < usable (both compressed with the same theta,
 * Montgomery form); reported as spb_nonzero_rows_dev reports. The table's usable rows are sorted in the workspace of
 * spb_permute_expression_pair_dev, so the check needs no more device memory than that call. */
int spb_lookup_missing_rows_dev(spb_ctx* ctx, const spb_fr* d_input, const spb_fr* d_table, size_t usable, uint32_t cap, uint32_t* rows_out, uint64_t* total_out);
/* Copy constraints of n_cols permutation columns over n = 2^k rows (HOST arrays of device pointers to their Lagrange values and
 * sigma columns). For every column c and row i < usable, the cell (c', i') that sigma_c[i] = delta^c' omega^i' labels must hold
 * the same value as (c, i). For column c, cells_out[4 (c cap + m) ..] = (c, i, c', i') of its m-th failing row, m < min(cap,
 * totals_out[c]), and totals_out[c] = its number of failing rows. A sigma entry of a usable row that labels no cell of a
 * usable row (c' >= n_cols or i' >= usable) is a malformed key: SPB_ERR_DATA, and the error text names the column and row
 * of the first such entry (lowest column, then lowest row); the outputs are then only the zeroed totals. usable <= 2^k. */
int spb_copy_mismatches_dev(spb_ctx* ctx, uint32_t k, const spb_fr* const* d_values, const spb_fr* const* d_sigma, uint32_t n_cols, size_t usable, uint32_t cap,
                            uint32_t* cells_out, uint64_t* totals_out);

/* ---- proving-key check ([UPSTREAM] halo2_proofs/src/plonk.rs ProvingKey::read in SerdeFormat::RawBytes, and
 * permutation::keygen::Assembly) ---------------------------------------------------------------------------------------
 * Inputs are device buffers of the context's first device and are not written; outputs are HOST values, filled before the call
 * returns. A NULL context, or a NULL pointer the call would read or write, is SPB_ERR_ARG.
 * Kernel launches (spb_kernel_launches): spb_fr_first_noncanonical_dev 1 (0 when n = 0); spb_sigma_check_dev 7 per column,
 * less 2 per column when usable = 2^k (no blinding rows) and 2 per column when usable = 0 (0 when n_cols = 0). */
/* *first_out = the lowest index i < n whose stored limbs, read as a 256-bit integer, are >= r (halo2curves' from_raw_bytes
 * rejects them); n when every element is canonical. Used on each polynomial of a .pkey right after it lands in device memory. */
int spb_fr_first_noncanonical_dev(spb_ctx* ctx, const spb_fr* d, size_t n, uint64_t* first_out);
/* Is sigma (n_cols HOST-held device pointers, 2^k rows each) a permutation of the cells (c, i), c < n_cols, i < 2^k, of the kind
 * permutation::keygen::Assembly builds? sigma_c[i] = delta^c' omega^i' labels the cell (c', i'). Three kinds of failure q, for
 * each column c: totals_out[3 c + q] = their exact number, rows_out[(3 c + q) cap + m] = the m-th row, ascending, m < min(cap,
 * total):
 *   q = 0 (label):      rows i < usable whose sigma_c[i] labels no cell of a usable row (no column c' < n_cols, or i' >= usable);
 *   q = 1 (blinding):   rows i >= usable whose sigma_c[i] is not their own label delta^c omega^i (Assembly::copy refuses rows
 *                       >= usable, so they are fixed points);
 *   q = 2 (unlabelled): cells (c, i), i < 2^k, that no sigma entry of any column labels.
 * All totals zero: as many entries as cells, each labels a cell and every cell is labelled, so sigma is a bijection of the cells
 * that fixes the blinding rows. Each entry is decoded once (a fixed point needs no decode) and its cell marked in an
 * n_cols 2^k-bit map; the report does not depend on the order of the device's atomics. usable <= 2^k, k <= 28. */
int spb_sigma_check_dev(spb_ctx* ctx, uint32_t k, const spb_fr* const* d_sigma, uint32_t n_cols, size_t usable, uint32_t cap, uint32_t* rows_out,
                        uint64_t* totals_out);

/* ---- argument provers, device resident ([UPSTREAM] halo2_proofs/src/plonk/{permutation,lookup}/prover.rs) ----------- */
/* permutation::Argument::commit for ONE set (a chunk of <= degree-2 columns, first_col = its index of first column in
 * the permutation): over all n = 2^k rows
 *   d_z[0] = *last_z,  d_z[i+1] = d_z[i] * prod_c (v_c[i] + beta*delta^(first_col+c)*omega^i + gamma) / prod_c (v_c[i] + beta*sigma_c[i] + gamma)
 * then the last n_blinds entries are overwritten with `blinds` (the caller's RNG draws, in order) and
 * *last_z <- d_z[n - n_blinds - 1]. d_values / d_sigma: HOST arrays of n_cols device pointers (Lagrange basis). */
int spb_permutation_product_dev(spb_ctx* ctx, uint32_t k, const spb_fr* const* d_values, const spb_fr* const* d_sigma, uint32_t n_cols, uint32_t first_col,
                                const spb_fr* beta, const spb_fr* gamma, const spb_fr* blinds, uint32_t n_blinds, spb_fr* last_z, spb_fr* d_z);
/* lookup Permuted::commit_product: d_z[0] = 1, d_z[i+1] = d_z[i] * (a[i]+beta)(s[i]+gamma) / ((a'[i]+beta)(s'[i]+gamma)),
 * last n_blinds entries <- blinds. a, s = compressed input / table; a', s' = their permuted forms (all n rows). */
int spb_lookup_product_dev(spb_ctx* ctx, size_t n, const spb_fr* d_compressed_input, const spb_fr* d_compressed_table, const spb_fr* d_permuted_input,
                           const spb_fr* d_permuted_table, const spb_fr* beta, const spb_fr* gamma, const spb_fr* blinds, uint32_t n_blinds, spb_fr* d_z);
/* d_out[i] = sum_p weights[p] * d_polys[p][i] (weights: host array). */
int spb_weighted_sum_dev(spb_ctx* ctx, const spb_fr* const* d_polys, const spb_fr* weights, size_t count, spb_fr* d_out, size_t n);

/* ---- SHPLONK multi-open prover ([UPSTREAM] halo2_proofs/src/poly/kzg/multiopen/shplonk/prover.rs) ------------------- */
/* One rotation set as construct_intermediate_sets (shplonk.rs) yields it: the polynomials opened at exactly `points`,
 * in first-queried order, with evals[j * n_points + p] = poly_j(points[p]). Polynomials are device pointers in
 * coefficient form, n coefficients each. */
typedef struct {
  const spb_fr* points;
  uint32_t n_points;             /* 1..8 */
  const spb_fr* const* d_polys;  /* host array of n_polys device pointers */
  uint32_t n_polys;
  const spb_fr* evals;
} spb_rotation_set;
typedef struct spb_shplonk spb_shplonk;
/* After squeezing y and v: h(X) = sum_i v^i * [sum_j y^j (P_ij(X) - R_ij(X))] / Z_{S_i}(X), committed with
 * `g`; the handle keeps h(X) on the device until the second call. The caller's polynomials must stay alive and
 * unchanged until then. */
int spb_shplonk_begin_dev(spb_ctx* ctx, const spb_srs* srs, size_t n, const spb_rotation_set* sets, uint32_t n_sets, const spb_fr* y, const spb_fr* v,
                          spb_g1* h_commitment, spb_shplonk** out);
/* After squeezing u: L(X) = sum_i v^(s-1-i) Z_{T\S_i}(u) sum_j y^(m_i-1-j) (P_ij(X) - R_ij(u)) - Z_T(u) h(X); commits
 * L(X) / (X - u) / Z_{T\S_0}(u). Consumes the handle (also on error, a null argument included). */
int spb_shplonk_finish_dev(spb_ctx* ctx, spb_shplonk* s, const spb_fr* u, spb_g1* commitment);
/* Releases an open handle without finishing it (a caller that fails between the two calls). While a handle is open the
 * context's SHPLONK workspace is held: a second handle allocates its own buffers, and spb_release_workspace fails. */
void spb_shplonk_abort(spb_ctx* ctx, spb_shplonk* s);

/* ---- BN254 pairing ([UPSTREAM] halo2curves src/bn256/engine.rs: multi_miller_loop, final_exponentiation; reached by
 * halo2's KZG verifier, poly/kzg/strategy.rs) ------------------------------------------------------------------------------ */
/* A G2 affine point as the params file's G2 trailer stores it: x.c0, x.c1, y.c0, y.c1 (Fq2 = Fq[u]/(u^2 + 1)), Montgomery
 * limbs; the identity is (0, 0). A Gt value: the 12 Fq coefficients of Fq12 in halo2curves' order c0.c0.c0, c0.c0.c1, ...,
 * c1.c2.c1 (tower Fq6 = Fq2[v]/(v^3 - (9 + u)), Fq12 = Fq6[w]/(w^2 - v)), Montgomery limbs. */
typedef struct { spb_fq x[2], y[2]; } spb_g2_affine;
typedef struct { spb_fq c[12]; } spb_gt;
/* *out = prod_i e(p[i], q[i]) for the optimal ate pairing e: the product of the Miller values raised to (p^12 - 1) / r, so a
 * pairing equals upstream's `Bn256::pairing`. A pair in which either point is the identity contributes one; n = 0 gives one.
 * Every input is checked on the device first: G1 points as the checked params read checks them (coordinates below p, on
 * y^2 = x^3 + 3, or the identity), G2 points likewise on the twist y^2 = x^3 + 3/(9+u) and in the order-r subgroup ([r]Q = O).
 * The first invalid input in the order p[0], q[0], p[1], q[1], ... gives SPB_ERR_DATA with its name, index and reason in the
 * error text, e.g. "q[17]: not in the r-torsion subgroup" or "p[3]: not on the curve", and *out is untouched.
 * One launch sequence on the context's first device (also when it lists several): the check, one Miller-loop thread per pair,
 * one final-exponentiation thread; 3 kernel launches (spb_kernel_launches) whatever n. Synchronous: the stream contract of
 * the host-buffer entry points; spb_last_device_ms gives the device time of the three kernels. NULL context or out, or NULL
 * p / q with n > 0: SPB_ERR_ARG. The first call makes the CUDA context reserve the kernels' per-thread stacks for every thread
 * the GPU can hold (826 MiB on an H100 80GB HBM3), which the context keeps until it is destroyed. */
int spb_pairing(spb_ctx* ctx, const spb_g1_affine* p, const spb_g2_affine* q, size_t n, spb_gt* out);
/* n_checks independent pairing checks in one launch sequence: ok[j] = 1 iff prod_{i<m} e(p[j*m+i], q[j*m+i]) == 1, else 0.
 * A KZG opening is one check of m = 2 pairs, e(P1, [1]_2) e(P2, -[s]_2) = 1; a batch of proofs gets one verdict per proof.
 * Inputs are checked as in spb_pairing over all m * n_checks pairs (SPB_ERR_DATA naming the first invalid one, ok untouched);
 * then one Miller-loop thread per pair and one final-exponentiation thread per check: 3 kernel launches whatever m and
 * n_checks. m = 0 gives ok[j] = 1 for every check without touching the device; n_checks = 0 does nothing. NULL context, NULL
 * ok with n_checks > 0, or NULL p / q with m n_checks > 0: SPB_ERR_ARG. spb_last_device_ms as for spb_pairing. */
int spb_pairing_check_batch(spb_ctx* ctx, const spb_g1_affine* p, const spb_g2_affine* q, size_t m, size_t n_checks, int32_t* ok);

/* ---- test / bench utilities -------------------------------------------------------------------------------- */
/* out[i] = scalars[i] * G1 (affine), computed on the device */
int spb_g1_fixed_base_mul(spb_ctx* ctx, const spb_fr* scalars, size_t n, spb_g1_affine* out);
/* The host-side scheduling pass spb_graph_evaluate_dev applies to a program before it runs it (one-part Horner steps placed next to
 * the calculation that produces the part; intermediates renamed to scratch slots by liveness -- csrc/quotient.cu), without any
 * device work: out_words receives the rescheduled program (same encoding, targets = slots < *num_slots). Returns SPB_ERR_STATE
 * when the pass declines (malformed program, a target written twice): the caller's program is then run as it is. */
int spb_test_schedule_program(const uint32_t* program, size_t program_words, uint32_t num_calculations, uint32_t* out_words, size_t out_capacity,
                              size_t* out_count, uint32_t* num_slots, uint32_t* out_calculations);
/* Elementwise device field arithmetic for parity tests of csrc/field.cuh, on raw limbs (field 0 = Fr, 1 = Fq; an Fq element
 * travels as an spb_fr). Binary: op 0 mul, 1 add, 2 sub. Unary, b unread: 3 sqr, 4 neg, 5 dbl, 6 inv, 7 to_mont, 8 from_mont,
 * 9 is_canonical (out = 1 or 0 in limb 0). Powers: 10 pow (exponent b as a canonical 256-bit integer), 11 pow_u64 (exponent the
 * low 64 bits of b). b must be readable for every op. */
int spb_test_field_op(spb_ctx* ctx, int field, int op, const spb_fr* a, const spb_fr* b, spb_fr* out, size_t n);
/* out[i] = a[i] * b[i] - c[i] * d[i] through fp_mul_sub_mul (two products under one Montgomery reduction). */
int spb_test_field_mul_sub_mul(spb_ctx* ctx, int field, const spb_fr* a, const spb_fr* b, const spb_fr* c, const spb_fr* d, spb_fr* out, size_t n);
/* Elementwise G1 operations of csrc/curve.cuh for parity tests. p, q and out hold n points of four spb_fr each, XYZZ
 * {x, y, zz, zzz} in Montgomery Fq; an affine operand is the (x, y) of its slot. op 0: p + q (q affine, xyzz_add_mixed);
 * 1: p + q (xyzz_add); 2: 2p (xyzz_dbl); 3: 2p (p affine, xyzz_dbl_affine); 4: p in affine (out = {x, y, 0, 0}); 5: k[i] * p
 * (xyzz_mul_u32; k may be NULL for the other ops); 6: affine_check of p's (x, y) (out x limb 0 = the verdict: 0 valid,
 * 1 x not canonical, 2 y not canonical, 3 off the curve). q must be readable for every op. */
int spb_test_curve_op(spb_ctx* ctx, int op, const spb_fr* p, const spb_fr* q, const uint32_t* k, spb_fr* out, size_t n);
/* modular-multiply throughput microbenchmark: `iters` dependent products per thread over `threads` threads, `ilp`
 * independent chains each (1, 2 or 4; ilp | 0x100 = two chains of squarings); returns device milliseconds in *ms. */
int spb_bench_modmul(spb_ctx* ctx, int field, uint32_t threads, uint32_t iters, int ilp, float* ms);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif
