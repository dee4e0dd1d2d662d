/*
 * gccnmf_b200 -- C ABI of the H100-native (sm_90a) GCC-NMF separation hot path.
 *
 * The reference (seanwood/gcc-nmf) has no FFI: its boundary is the Python call surface of
 * gccNMF/gccNMFFunctions.py, gccNMF/librosaSTFT.py and gccNMF/realtime/gccNMFProcessor.py.
 * Each entry point below is the device-side replacement of one of those Python functions
 * (cited per function as file:line relative to the reference root) and is what a ctypes
 * binding in the reference would call (see INTEGRATION.md).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless its name ends in `_host`;
 *  - the caller owns all buffers (including workspaces, sized by the *_workspace_bytes helpers);
 *    the library borrows them for the duration of the call and never frees them;
 *  - every call is asynchronous on `stream` (a cudaStream_t passed as void*; NULL = legacy default
 *    stream) and returns 0 on success or a negative gccnmf_status; no C++ exception crosses the ABI;
 *  - array layouts are the reference's numpy C-order layouts: spectrograms (channel, F, T) with T
 *    contiguous, W (F, K), H (K, 2T), masks (S, K, T), signals (S, 2, n);
 *  - complex64 is interleaved (re, im) float pairs, complex128 interleaved double pairs;
 *  - a handle is bound to one device and is not thread-safe (use one per host thread / stream).
 */
#ifndef GCCNMF_B200_H_
#define GCCNMF_B200_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define GCCNMF_API __attribute__((visibility("default")))
#else
#define GCCNMF_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define GCCNMF_ABI_VERSION 2

typedef struct gccnmf_handle gccnmf_handle;

typedef enum gccnmf_status {
  GCCNMF_OK = 0,
  GCCNMF_ERR_INVALID_ARGUMENT = -1, /* librosaSTFT.ParameterError / ValueError in the reference   */
  GCCNMF_ERR_CUDA = -2,             /* a CUDA runtime call failed; text in gccnmf_last_error       */
  GCCNMF_ERR_WORKSPACE = -3,        /* workspace pointer NULL or too small                          */
  GCCNMF_ERR_UNSUPPORTED = -4,      /* shape outside what the kernels were built for               */
  GCCNMF_ERR_NO_DEVICE = -5         /* no CUDA device: there is NO CPU fallback                     */
} gccnmf_status;

/* ---- handle ------------------------------------------------------------------------------- */
GCCNMF_API int gccnmf_abi_version(void);
/* Binds to `device`; fails with GCCNMF_ERR_NO_DEVICE when no GPU is visible. */
GCCNMF_API int gccnmf_create(gccnmf_handle** out, int device);
GCCNMF_API int gccnmf_destroy(gccnmf_handle* h);
/* Text of the last error recorded on this handle (never NULL; h may be NULL for create errors). */
GCCNMF_API const char* gccnmf_last_error(const gccnmf_handle* h);
GCCNMF_API const char* gccnmf_status_string(int status);
/* Count of kernels this handle has launched since creation (bench.py's `gpu_launches`). */
GCCNMF_API int64_t gccnmf_launch_count(const gccnmf_handle* h);
/* Options (A/B switches between sm_90a code paths of this library; all ranks of a sharded run must use the same ones so
 * that W stays bit-identical).  Defaults in brackets.
 *   "force_simt_nmf" [0]        KL-NMF contractions on the float32 SIMT kernels even where the wgmma plane GEMM applies
 *   "nmf_pdl" [1]               programmatic dependent launch between the kernels of a KL-NMF iteration
 *   "gemm_cluster" [-1]         plane GEMM cluster shape 10 CN + CM (11, 12, 21, 22) instead of the automatic choice
 *   "argmax_refine_shared" [1]  float64 refinement of near-tie argmax decisions with E staged in shared memory
 *   "argmax_persistent" [1]     all-TDOA argmax GEMM as one persistent CTA per SM (epilogue from registers); 0 = one CTA per tile
 *   "wh_tile" [0]               tile width of the W.H contractions (104 / 112 / 120 / 128 / 256) instead of the planned one
 *   "gemm_pair" [-1]            plane GEMM on CTA pairs (1 x 2 clusters sharing the B tile): -1 where a call site prefers it, 0 never, 1 wherever possible
 *                               (bit-identical results either way)
 *   "l2_persist" [0]            KL-NMF loop: persisting L2 access-policy window over G^T (1 = float32 master, 2 = master + planes)
 *   "wh_split2" [0]             W.H contractions as plain 128 x 208 tiles with the contraction split in two halves that a
 *                               (1, 1, 2) cluster sums through distributed shared memory
 *   "w_cluster_reduce" [1]      W-update numerator: k-splits summed inside (1, 1, splits) clusters where every cluster of the
 *                               launch is resident at once (else k-split slabs)
 *   "mc_light_signal" [1]       sharded runs: arrival signal as device-scope fence + relaxed red (0: MEMBAR.SYS + release)
 *   "pull_force_pack" [0]       pull exchange: always through the pack kernel (diagnostics)
 *   "gemm_preload" [1]          bit 0: the W.H ratio epilogue fetches V during the main loop
 *   "gemm_streaming" [0]        st.global.cs / ld.global.cs for the k-split partials of the W-update numerator */
GCCNMF_API int gccnmf_set_option(gccnmf_handle* h, const char* name, int value);

/* ---- a1: STFT  (gccNMF/librosaSTFT.py:20-181 via gccNMFFunctions.py:61-67) ------------------ */
/* Frame count 1 + (num_samples - n_fft) / hop (librosaSTFT.py:425); <1 -> GCCNMF_ERR_INVALID_ARGUMENT. */
GCCNMF_API int gccnmf_stft_num_frames(int64_t num_samples, int n_fft, int hop);
/*
 * samples (channels, num_samples) f32 with row stride `sample_stride`; window (n_fft) f64 on device;
 * X (channels, F, T) c64.  Computation is float64 like the reference (window f64 * frame, double FFT)
 * and rounded once to complex64.  conjugate != 0 reproduces librosaSTFT.py:179 (offline path);
 * conjugate == 0 is numpy.fft.rfft (online / real-time path, onlineSpeechEnhancement.ipynb:410).
 * V (F, channels*T) f32 = |X| with the channels concatenated in time (runGCCNMF.py:40); may be NULL.
 * channels must be 1 or 2; n_fft a power of two in [32, 4096].
 */
GCCNMF_API int gccnmf_stft(gccnmf_handle* h, const float* samples, int64_t sample_stride, int channels,
                int64_t num_samples, const double* window, int n_fft, int hop, int conjugate,
                float* X, float* V, void* stream);

/* ---- a9: iSTFT + overlap-add  (librosaSTFT.py:183-286 via gccNMFFunctions.py:153-163) ------- */
/* Output length per signal: n_fft + hop (T-1) - (center ? n_fft : 0). */
GCCNMF_API int64_t gccnmf_istft_length(int n_fft, int hop, int T, int center);
GCCNMF_API size_t gccnmf_istft_workspace_bytes(int batch, int n_fft, int T);
/*
 * spec (batch, F, T) c64 -> y (batch, length) f32.  Per frame: Hermitian rebuild from conj(col)
 * (librosaSTFT.py:278), single-precision inverse FFT (:279), real part times window (f64),
 * sequential float32 overlap-add in frame order (:281), optional centre trim (:283-284), times
 * `gain` (gccNMFFunctions.py:155,163).  conjugate == 0 skips the conj (numpy.fft.irfft convention).
 */
GCCNMF_API int gccnmf_istft_ola(gccnmf_handle* h, const float* spec, int batch, int n_fft, int hop, int T,
                     const double* window, float gain, int center, int conjugate, float* y,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ---- a2: KL-NMF  (gccNMFFunctions.py:69-83) -------------------------------------------------- */
GCCNMF_API size_t gccnmf_klnmf_workspace_bytes(int F, int T2, int K);
/* 1 when the contractions of this shape run on the tensor cores (wgmma, TMA-fed plane GEMM over bf16 hi/lo operand planes: K % 8 == 0, K >= 32,
 * F, T2 >= 128), 0 when they run on the float32 SIMT kernels (small or odd shapes, or GCCNMF_NMF_PATH=simt). */
GCCNMF_API int gccnmf_klnmf_uses_tensor_cores(const gccnmf_handle* h, int F, int T2, int K);
/*
 * V (F, T2) f32 non-negative; W (F, K) and H (K, T2) f32 hold the initial values on entry (the
 * seeded numpy draw of gccNMFFunctions.py:70-73 is made on the host) and the result on return.
 * Runs `iterations` passes of lines :76-81 (H update, W update on the recomputed W.H, unit-L2 atoms).
 * update_W == 0 runs only the H update (:76) with a fixed dictionary (the undefined
 * inferCoefficientsKLNMF of onlineSpeechEnhancement.ipynb:433).
 */
GCCNMF_API int gccnmf_klnmf(gccnmf_handle* h, const float* V, int F, int T2, float* W, float* H, int K,
                 int iterations, float sparsity_alpha, float epsilon, int update_W,
                 void* workspace, size_t workspace_bytes, void* stream);
/*
 * B clips of one shape (F, T2, K) in one call: clip b's W and H come out bit for bit as gccnmf_klnmf on that clip alone would
 * leave them (same handle, same options).  Clip b's V is read in place at V + b * clip_stride_v with row pitch ld_v (>= T2):
 * a contiguous (B, F, T2) stack is ld_v = T2, clip_stride_v = F * T2; clips side by side in the columns of one (F, B T2) matrix
 * are ld_v = B T2, clip_stride_v = T2.  W (B, F, K) and H (B, K, T2) are contiguous clip-major stacks holding the
 * initial values on entry and the results on return.  On the tensor-core path every launch of an iteration covers all clips; the
 * workspace grows linearly in B (B x gccnmf_klnmf_workspace_bytes at tensor-core shapes).  B is 1 .. 8191.
 */
GCCNMF_API size_t gccnmf_klnmf_batched_workspace_bytes(int B, int F, int T2, int K);
GCCNMF_API int gccnmf_klnmf_batched(gccnmf_handle* h, const float* V, int64_t ld_v, int64_t clip_stride_v, int B, int F, int T2,
                         float* W, float* H, int K, int iterations, float sparsity_alpha, float epsilon, int update_W,
                         void* workspace, size_t workspace_bytes, void* stream);
/*
 * B clips of different lengths in one call: clip b's W and H come out bit for bit as gccnmf_klnmf on that clip alone would leave
 * them (same handle, same options).  V, ld_v, T2 and H are HOST arrays of B entries, read only during the call (no pointer to them
 * is kept): clip b's V is (F, T2[b]) at V[b] with row pitch ld_v[b] >= T2[b], read in place (an STFT output view works); its H is
 * (K, T2[b]) contiguous at H[b].  W is a contiguous (B, F, K) stack.  W and H hold the initial values on entry and the results on
 * return.  On the tensor-core path each contraction of an iteration is launched once per distinct tile width among the clips' solo
 * plans, and each other kernel once for all clips; the launch count does not grow with B.  Clips the float32 SIMT path takes, and
 * clips under an option the batch form leaves out, run one at a time as gccnmf_klnmf_batched runs them.
 * Workspace (gccnmf_klnmf_ragged_workspace_bytes): a per-call table of 1280 B + 256 bytes, then clip b's region of a batched run on
 * its shape (gccnmf_klnmf_batched_workspace_bytes(1, F, T2[b], K), which is gccnmf_klnmf_workspace_bytes(F, T2[b], K) at
 * tensor-core shapes); nothing is padded to the longest clip.  The table is written by a stream-ordered copy from host memory
 * that the call owns.  B is 1 .. 8191; B, null pointers, T2[b] <= 0, ld_v[b] < T2[b], negative iterations and a short workspace
 * are refused before anything is enqueued.  The size function returns 0 for such arguments.
 */
GCCNMF_API size_t gccnmf_klnmf_ragged_workspace_bytes(int B, int F, const int* T2, int K);
GCCNMF_API int gccnmf_klnmf_ragged(gccnmf_handle* h, const float* const* V, const int64_t* ld_v, const int* T2, int B, int F,
                         float* W, float* const* H, int K, int iterations, float sparsity_alpha, float epsilon, int update_W,
                         void* workspace, size_t workspace_bytes, void* stream);
/*
 * Frame-sharded dictionary learning (multi-GPU; SURVEY.md section 8e).  A rank holds the columns V_s
 * (F, T2s), H_s (K, T2s) of its frames and a replica of W.  The loop of gccNMFFunctions.py:75-81 becomes
 *
 *   gccnmf_klnmf_begin(...)                       once (operand re-layout for the tensor-core path)
 *   for it in range(iterations):
 *       gccnmf_klnmf_step_numer(..., it, numer)   H_s update (:76); numer = [ (V_s/(W H_s)).H_s^T (F*K) | rowsum(H_s) (K) ]
 *       all-reduce(sum) of numer over the ranks   ONE collective of F*K + K floats per iteration
 *       gccnmf_klnmf_step_apply(..., numer)       W *= numer / rowsum (:77), unit-L2 atoms (:79-80), H_s *= norms (:81)
 *   gccnmf_klnmf_end(..., iterations)             materialises the last (lazily applied) H_s rescale
 *
 * All state lives in W, H and the caller-owned workspace (gccnmf_klnmf_workspace_bytes), which must not be
 * touched between begin and end.  Every rank computes a bit-identical W from the same all-reduced numer.
 */
GCCNMF_API int gccnmf_klnmf_begin(gccnmf_handle* h, const float* V, int F, int T2, const float* W, const float* H,
                       int K, void* workspace, size_t workspace_bytes, void* stream);
GCCNMF_API int gccnmf_klnmf_step_numer(gccnmf_handle* h, const float* V, int F, int T2, const float* W, float* H,
                            int K, float sparsity_alpha, float epsilon, int iteration, float* numer,
                            void* workspace, size_t workspace_bytes, void* stream);
GCCNMF_API int gccnmf_klnmf_step_apply(gccnmf_handle* h, int F, int T2, float* W, float* H, int K,
                            const float* numer, void* workspace, size_t workspace_bytes, void* stream);
/*
 * Fused collective variant of step_apply for NVSwitch systems: every rank's step_numer wrote its partial into the
 * SAME offset of a symmetric buffer bound to an NVLink multicast object; `numer_multicast` is the multicast address
 * of that buffer.  After a cross-rank barrier the W update reads each numerator / row-sum word with
 * multimem.ld_reduce.add.f32 -- the sum over ranks is formed inside the switch (NVLS) while the kernel streams it,
 * so there is no separate all-reduce kernel and no second pass over the 2 MB.  Every rank receives the same
 * switch-reduced value, hence a bit-identical W.  Tensor-core path only (GCCNMF_ERR_UNSUPPORTED otherwise).
 */
GCCNMF_API int gccnmf_klnmf_step_apply_multimem(gccnmf_handle* h, int F, int T2, float* W, float* H, int K,
                                     const float* numer_multicast, void* workspace, size_t workspace_bytes,
                                     void* stream);
/* One iteration of a frame-sharded run with the cross-rank exchange fused into the kernels: the numerator pack signals "this rank
 * is complete" to every rank with one multimem.red on an arrival counter, the W-update kernel waits on its own copy of the counter
 * and reads the sum over ranks with multimem.ld_reduce (formed inside the NVSwitch) -- no host-launched barrier, no all-reduce.
 * numer_local / counter_local: this rank's addresses inside its symmetric buffer ((F*K + K) floats + one uint32 per buffer);
 * numer_multicast / counter_multicast: the NVLink multicast addresses of the same offsets; arrivals_expected = world size x the
 * number of times this buffer has been used so far (including this one).  Double-buffer by iteration parity. */
GCCNMF_API int gccnmf_klnmf_step_multimem(gccnmf_handle* h, const float* V, int F, int T2, float* W, float* H, int K,
                               float sparsity_alpha, float epsilon, int iteration, float* numer_local,
                               const float* numer_multicast, const uint32_t* counter_local, uint32_t* counter_multicast,
                               uint32_t arrivals_expected, void* workspace, size_t workspace_bytes, void* stream);
/* The same iteration with a TWO-SHOT exchange: after the pack every rank sums only its 1 / world slice of the numerator with
 * multimem.ld_reduce and multicasts the sum into the `reduced` buffer of every rank (multimem.st); the W update reads its local
 * `reduced` copy once the second arrival counter is complete.  Link traffic per GPU and iteration: one numerator out, one in, for any
 * world size (the one-shot form above makes every GPU serve `world` numerators).  numer_* / reduced_*: two symmetric buffers of
 * (F*K + K) floats (local and multicast addresses); counters_*: two consecutive uint32 in symmetric memory (pack arrivals, slice
 * arrivals), zero before the first iteration; arrivals_expected = world x (iteration + 1).  No double buffering needed: a rank
 * re-packs only after its own W update, which waits for every rank's slice. */
GCCNMF_API int gccnmf_klnmf_step_multimem2(gccnmf_handle* h, const float* V, int F, int T2, float* W, float* H, int K,
                                float sparsity_alpha, float epsilon, int iteration, int rank, int world, float* numer_local,
                                const float* numer_multicast, const float* reduced_local, float* reduced_multicast,
                                const uint32_t* counters_local, uint32_t* counters_multicast, uint32_t arrivals_expected,
                                void* workspace, size_t workspace_bytes, void* stream);
/* PULL exchange (the default of the sharded pipeline): nothing is pushed over the links and nothing is reduced in the switch.  The
 * numerator contraction writes this rank's (F, K) partial straight into its symmetric buffer and its last CTA adds 1 to every rank's
 * arrival counter (device-scope fence + relaxed red: the published data is local, peers fetch it through this GPU's L2); then
 *   two_shot = 2: the exchange happens INSIDE the W update, tile by tile: the CTA that owns a 32 x 128 tile of U sums this rank's
 *                 k-split slabs for it, publishes the tile in the symmetric buffer, flags it on every rank, waits for the same tile
 *                 of the other ranks and reads them with plain peer loads -- five launches per iteration, like the single-GPU loop;
 *   two_shot = 0: every rank's W update reads all ranks' partials with plain peer loads, added in rank order;
 *   two_shot = 1: each rank first sums its 1 / world slice that way into its own buffer, signals, and the W updates fetch each word
 *                 from its owner -- one numerator in each direction per GPU for any world size.
 * Row sums of G are read from every rank's slots.  bases: HOST array of `world` device pointers, every rank's buffer as mapped in
 * this process (gccnmf_klnmf_pull_buffer_floats(F, layout_T2, K) floats each, zero before the first iteration; layout_T2 = the
 * largest 2T over the ranks; epoch = iterations earlier runs executed on this buffer: the arrival counters keep counting).  Needs the
 * cluster-reduced numerator contraction for direct = 1 (see gccnmf_klnmf_pull_supported). */
GCCNMF_API int64_t gccnmf_klnmf_pull_buffer_floats(int F, int layout_T2, int K);
/* Bit mask.  0: gccnmf_klnmf_step_pull does not cover this shard shape on this device.  Bit 0: it does, through the pack kernel
 * (k-split slabs and row-sum slots summed into the symmetric buffer, then the signal).  Bit 1: also in the direct form (the numerator
 * contraction sums its k-splits inside clusters, writes the buffer itself and signals from its last CTA): `direct` of step_pull must be
 * the same on every rank, 1 only if every rank has this bit.  Bit 2: form 2 (exchange inside the W update) is available: every tile
 * CTA of the W update is resident at once. */
GCCNMF_API int gccnmf_klnmf_pull_supported(gccnmf_handle* h, int F, int T2, int K);
GCCNMF_API int gccnmf_klnmf_step_pull(gccnmf_handle* h, const float* V, int F, int T2, float* W, float* H, int K,
                           float sparsity_alpha, float epsilon, int iteration, int64_t epoch, int rank, int world,
                           void* const* bases, int layout_T2, int two_shot, int direct, void* workspace, size_t workspace_bytes,
                           void* stream);
GCCNMF_API int gccnmf_klnmf_end(gccnmf_handle* h, int F, int T2, float* W, float* H, int K, int iterations_done,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ---- a3 + a4: PHAT coherence and angular spectrogram  (runGCCNMF.py:44, gccNMFFunctions.py:85-92) */
/*
 * X (2, F, T) c64; expJOmegaTau (F, D) c128 = exp(-2 pi i f tau) built on the host in float64
 * exactly as gccNMFFunctions.py:89.  coherence (F, T) c64 = X0 conj(X1) / |X0| / |X1| (unguarded,
 * 0/0 -> NaN); angular (D, T) f64 = sum_f Re(coherence * E); mean_angular (D) f64 = mean over T
 * (runGCCNMF.py:46).  coherence, angular and mean_angular may each be NULL.
 * x_is_coherence != 0: X is an already-normalised (F, T) coherence (the argument
 * gccNMFFunctions.getAngularSpectrogram takes, :85) and is used as is.
 */
GCCNMF_API size_t gccnmf_phat_angspec_workspace_bytes(int F, int T, int D);
GCCNMF_API int gccnmf_phat_angspec(gccnmf_handle* h, const float* X, int F, int T, int x_is_coherence,
                        const double* expJOmegaTau, int D, float* coherence, double* angular, double* mean_angular,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---- a6 / a10 / a11: GCC-NMF per TDOA  (gccNMFFunctions.py:118-135; offlineSpeechEnhancement.ipynb:444-450) */
/*
 * gccnmf[d, k, t] = sum_f Re(coherence[f, t] * E[f, d]) * W[f, k] accumulated in float64
 * (the reference contracts in complex128 / float64).  E (F, D) c128 holds either the selected
 * target TDOA columns (a6: D = number of targets) or all hypothesis TDOAs (a10/a11).
 * values (D, K, T) f32 (a6's output dtype, gccNMFFunctions.py:131) and/or argmax (K, T) int32 over d
 * with numpy.argmax semantics (first maximum; NaN counts as maximum).  Either may be NULL.
 */
GCCNMF_API int gccnmf_tdoa_gccnmf(gccnmf_handle* h, const float* coherence, int F, int T, const double* E,
                       int D, const float* W, int K, float* values, int32_t* argmax, void* stream);

/*
 * a10 / a11 fast path: argmax over ALL hypothesis TDOAs without materialising (K, D, T) float64.
 * For D a power of two in [8, 128], K % 8 == 0, K >= 64 the contraction runs as a wgmma GEMM over bf16 hi/lo planes of
 * Re(C E) (persistent kernel, float32 register accumulators) whose epilogue keeps the best / second-best value per (atom, frame) and the
 * candidates within the margin; every decision whose margin is inside the GEMM's worst-case
 * error is recomputed exactly in float64, so the result equals gccnmf_tdoa_gccnmf's argmax (the
 * reference's numpy.argmax on float64) on every input.  Other shapes run the float64 kernel directly.
 * *overflow_flag (device int32, may be NULL) receives the number of refined decisions; if it exceeds
 * gccnmf_tdoa_argmax_refine_capacity(K, T) the caller must recompute with gccnmf_tdoa_gccnmf.
 */
GCCNMF_API size_t gccnmf_tdoa_argmax_workspace_bytes(int F, int T, int D, int K);
GCCNMF_API int gccnmf_tdoa_argmax_refine_capacity(int K, int T);
GCCNMF_API int gccnmf_tdoa_argmax(gccnmf_handle* h, const float* coherence, int F, int T, const double* E, int D,
                       const float* W, int K, int32_t* argmax, int32_t* overflow_flag, void* workspace,
                       size_t workspace_bytes, void* stream);

/* ---- a7: coefficient masks  (gccNMFFunctions.py:137-143; offlineSpeechEnhancement.ipynb:466-472) */
/* nanargmax over S -> one-hot (S, K, T) f32.  *all_nan_flag (device int32, may be NULL) is set to 1
 * when some (k, t) is NaN for every target (numpy.nanargmax raises ValueError there). */
GCCNMF_API int gccnmf_coeff_mask(gccnmf_handle* h, const float* gccnmfs, int S, int K, int T, float* masks,
                      int32_t* all_nan_flag, void* stream);
/* mask[k, t] = lut[argmax[k, t]] with lut (D) u8 built on the host in float64 from
 * |tdoa[argmax] - tdoa[target]| < window (ipynb:468-471). */
GCCNMF_API int gccnmf_argmax_mask(gccnmf_handle* h, const int32_t* argmax, int K, int T, const uint8_t* lut,
                       int D, float* mask, void* stream);

/* ---- a11 / a13: online localisation, atom masks, Wiener-like filter ------------------------------
 * (notebooks/onlineSpeechEnhancement.ipynb:406-447, lowLatencySpeechEnhancement.ipynb:511-584,
 *  realtime/gccNMFProcessor.py:201-231,259-269).  The notebooks' frame loop carries one piece of state, the
 * accumulated maximum of the GCC-PHAT angular spectrum; it is a prefix maximum over time, so all frames are
 * processed in one batch. */
/* accumulated_max (D, T) f64 = running max over frames of angular (D, T); targets (T) i32 = its argmax over TDOA (:416-417). */
GCCNMF_API int gccnmf_online_targets(gccnmf_handle* h, const double* angular, int D, int T, double* accumulated_max,
                          int32_t* targets, void* stream);
/* mask (K, T) f32 from argmax (K, T) and the target TDOA index (per frame: targets (T) i32; or targets == NULL and
 * one float target_scalar, the Theano shared scalar of gccNMFProcessor.py:196).
 * mode 0 boxcar |argmax - target| < epsilon (ipynb:423-425; gccNMFProcessor.py:263);
 * mode 1 window exp(-(|argmax - target| / epsilon)^beta) / (1 + noise_floor) + noise_floor (gccNMFProcessor.py:265). */
GCCNMF_API int gccnmf_atom_mask(gccnmf_handle* h, const int32_t* argmax, int K, int T, const int32_t* targets,
                     float target_scalar, float epsilon, int mode, float beta, float noise_floor, float* mask,
                     void* stream);
/* Y (2, F, T) c64 = wiener * X with wiener (F, T) f32 = (W . mask) / rowsum(W) (ipynb:429-431,440;
 * gccNMFProcessor.py:267-269,209); wiener may be NULL when only Y is wanted. */
GCCNMF_API size_t gccnmf_wiener_apply_workspace_bytes(int F);
GCCNMF_API int gccnmf_wiener_apply(gccnmf_handle* h, const float* mask, const float* W, const float* X, int F, int T,
                        int K, float* Y, float* wiener, void* workspace, size_t workspace_bytes, void* stream);

/* ---- a8: masked reconstruction with mixture phase  (gccNMFFunctions.py:145-151) -------------- */
/* out[s, c] = (W . (H[:, c*T:(c+1)*T] * masks[s])) * exp(i angle(X[c])) ; out (S, 2, F, T) c64.
 * With a workspace of gccnmf_masked_recon_workspace_bytes the S x 2 products run on the tensor cores (the plane GEMM of the
 * KL-NMF loop over masked-H planes: 3 bf16 products per product, ~3e-6 relative); with workspace == NULL, or a shape the
 * tensor-core path does not cover, on the float32 SIMT kernel. */
GCCNMF_API size_t gccnmf_masked_recon_workspace_bytes(int S, int F, int T, int K);
GCCNMF_API int gccnmf_masked_recon_phase(gccnmf_handle* h, const float* masks, const float* X, const float* W,
                              const float* H, int S, int F, int T, int K, float* out, void* workspace,
                              size_t workspace_bytes, void* stream);

/* The numInferenceIterations > 0 branch of the notebooks' frame loop (onlineSpeechEnhancement.ipynb:433-440): with
 * H (K, 2T) f32 the inferred coefficients (channel c in columns [c T, (c + 1) T)),
 * wiener (2, F, T) f32 = (W . (H_c * mask)) / (W . H_c) and Y (2, F, T) c64 = wiener * X; wiener may be NULL. */
GCCNMF_API int gccnmf_wiener_apply_h(gccnmf_handle* h, const float* mask, const float* W, const float* H, const float* X, int F,
                          int T, int K, float* Y, float* wiener, void* stream);

/* ---- the whole offline path as one call ------------------------------------------------------------------
 * runGCCNMF.py:36-52 (num_targets >= 1: separation into num_targets sources) or the enhancement flow of
 * notebooks/offlineSpeechEnhancement.ipynb cells 12-41 (num_targets == 0: one target, all-TDOA argmax mask), every stage
 * enqueued on `stream` without a host synchronisation in between: the target TDOAs are picked by a device kernel with the
 * semantics of scipy.signal.argrelmax + the numSources largest peaks (gccNMFFunctions.py:94-116) and stay on the device. */
typedef struct gccnmf_pipeline_config {
  int window_size, hop_size;      /* N (= n_fft), hop                                                               */
  int num_tdoas, num_atoms;       /* D, K                                                                           */
  int num_iterations;             /* KL-NMF iterations                                                              */
  int num_targets;                /* S >= 1: separation; 0: enhancement (one target)                               */
  float sparsity_alpha, epsilon;  /* gccNMFFunctions.py:69                                                          */
  float target_window_seconds;    /* enhancement: |tdoa - tdoa[target]| < this (ipynb:468-471)                      */
} gccnmf_pipeline_config;
GCCNMF_API size_t gccnmf_pipeline_workspace_bytes(const gccnmf_pipeline_config* cfg, int64_t num_samples);
/* targets (num_targets) i32 ascending; *status |= 1 when the spectrum has fewer strict local maxima than num_targets. */
GCCNMF_API int gccnmf_pick_targets(gccnmf_handle* h, const double* mean_angular, int D, int num_targets, int32_t* targets,
                        int32_t* status, void* stream);
/* samples (2, n) f32; window (N) f64; E (F, D) c128; tdoas (D) f64; W (F, K), H (K, 2T) f32 in: seeded initial values
 * (gccNMFFunctions.py:70-73), out: learnt; signals (S, 2, gccnmf_istft_length(N, hop, T, 1)) f32; target_indexes (S) i32 and
 * status (1) i32 are device outputs: bit 0 too few peaks (the reference aborts), bit 1 all-NaN mask column (numpy raises),
 * bit 2 more near-tie argmax decisions than the float64 refinement list holds (re-run gccnmf_tdoa_gccnmf). */
GCCNMF_API int gccnmf_separate(gccnmf_handle* h, const gccnmf_pipeline_config* cfg, const float* samples, int64_t num_samples,
                    const double* window, const double* E, const double* tdoas, float* W, float* H, float* signals,
                    int32_t* target_indexes, int32_t* status, void* workspace, size_t workspace_bytes, void* stream);

/* ---- the offline path following a moving talker: targets per frame from a sliding window of the angular spectrogram -------
 * The sliding-window rule of realtime/gccNMFProcessor.py:219-226 (the real-time and low-latency engines' window), per frame of a
 * whole clip.  With A the (D, T) f64 angular spectrogram of gccnmf_phat_angspec and a window of w >= 1 frames:
 * - means[d][t] = the nanmean of A[d][t], A[d][t - 1], ..., A[d][max(0, t - w + 1)]: summed in float64 newest first, skipping
 *   NaN, divided by the number of non-NaN terms; NaN when all are NaN.  The window is cut at the start of the clip.  It is
 *   causal, so a target lags a move by up to w frames.
 * - targets[t] = the P largest strict interior local maxima of means[:, t], ascending (gccnmf_pick_targets' rule).  A frame with
 *   fewer than P peaks holds the targets of the latest earlier frame that had P, or floor((2 q + 1) D / (2 P)) before any such
 *   frame, and sets *status bit 0 (ORed in; the status is not cleared).
 * w < 1, P outside [1, D], D outside [3, 1024], T P >= 2^31 and NULL pointers are refused before anything is enqueued.
 * means may be NULL: the call then keeps them in a stream-ordered allocation (cudaMallocAsync) for its duration. */
GCCNMF_API int gccnmf_window_targets(gccnmf_handle* h, const double* angular, int D, int T, int window, int P, double* means,
                          int32_t* targets, int32_t* status, void* stream);
/* values (P, K, T) f32 = the float64 GCC-NMF contraction at P target TDOAs per frame, targets (T, P) i32 each in [0, D);
 * values[q][k][t] has the bits gccnmf_tdoa_gccnmf writes at (targets[t][q], k, t).  T P or P K T >= 2^31 is refused.
 * The targets are device data the call does not read on the host, and the kernel indexes E with them unchecked: a target outside
 * [0, D) is undefined behaviour (an out-of-bounds read of E).  gccnmf_window_targets only writes targets in [0, D). */
GCCNMF_API int gccnmf_target_gccnmf(gccnmf_handle* h, const float* coherence, int F, int T, const double* E, int D, const float* W,
                         int K, const int32_t* targets, int P, float* values, void* stream);
/* The enhancement mask with a target per frame: mask[k][t] = |tdoa[argmax[k][t]] - tdoa[targets[t]]| < window_seconds, in
 * float64 through a (D, D) u8 table built in lut_workspace (D * D bytes), whose row tau is the LUT of gccnmf_separate's
 * enhancement flow for target tau.  targets (T) i32; D <= 1024. */
GCCNMF_API int gccnmf_argmax_mask_frames(gccnmf_handle* h, const int32_t* argmax, int K, int T, const double* tdoas, int D,
                              const int32_t* targets, double window_seconds, uint8_t* lut_workspace, float* mask, void* stream);
/* gccnmf_separate with the targets of gccnmf_window_targets (P = num_targets, or 1 for the enhancement flow): one call, no host
 * synchronisation.  Separation: values at each frame's targets (gccnmf_target_gccnmf), then gccnmf_coeff_mask; source q is the
 * q-th target from the left in each frame.  Enhancement: gccnmf_argmax_mask_frames on the all-TDOA argmax.  frame_targets (T, S)
 * i32 and status (1) i32 are device outputs, window_means (D, T) f64 a device output that may be NULL.  Status bits as
 * gccnmf_separate's, except that bit 0 means a frame held earlier targets: information, not an error.  When every frame's targets
 * are gccnmf_separate's, the signals are gccnmf_separate's, byte for byte.  A window < 1, num_targets > num_tdoas, T S or S K T
 * >= 2^31, NULL pointers and a workspace smaller than gccnmf_pipeline_tracked_workspace_bytes are refused before anything is
 * enqueued.  The workspace size is 0 for a window < 1 or an invalid configuration. */
GCCNMF_API size_t gccnmf_pipeline_tracked_workspace_bytes(const gccnmf_pipeline_config* cfg, int localization_window, int64_t num_samples);
GCCNMF_API int gccnmf_separate_tracked(gccnmf_handle* h, const gccnmf_pipeline_config* cfg, int localization_window,
                            const float* samples, int64_t num_samples, const double* window, const double* E,
                            const double* tdoas, float* W, float* H, float* signals, int32_t* frame_targets,
                            double* window_means, int32_t* status, void* workspace, size_t workspace_bytes, void* stream);

/* ---- a13 + f-2: the real-time block path as one stream-ordered unit ----------------------------------
 * GCCNMFProcessor.processFrames (realtime/gccNMFProcessor.py:201-231 and the Theano graph of :245-270) with the
 * OverlapAddProcessor rings around it (realtime/utils.py:72-116) and, optionally, the per-frame coefficient inference of
 * notebooks/onlineSpeechEnhancement.ipynb:433-438.  Everything between the input block and the output block runs on
 * the device without a host synchronisation: five kernels per block (+ two per inference iteration), capturable in a
 * CUDA graph; the 8-block rings, the GCC-PHAT history, the sliding-window localisation and the target TDOA index are
 * device-resident state inside the caller-owned `state` buffer (sized by gccnmf_rt_state_bytes, filled by gccnmf_rt_init). */
typedef struct gccnmf_rt_config {
  int window_size;           /* N: power of two in [64, 2048] (config.py:63 windowSize)                              */
  int hop_size;              /* config.py:64                                                                          */
  int block_size;            /* samples per channel per audio block (config.py:65); the rings hold 8 blocks (utils.py:85) */
  int windows_per_block;     /* numTimePerChunk = blockSize // hopSize (config.py:112), at most 8                      */
  int num_atoms;             /* K                                                                                     */
  int num_tdoas;             /* D <= 128                                                                              */
  int history_length;        /* columns of the gccPHATHistory ring (runRealtimeGCCNMF.py:58)                          */
  int inference_iterations;  /* 0 = the reference's real-time class (numHUpdates is never used there); > 0: H-only KL updates */
  float sparsity_alpha;      /* of the inference updates (gccNMFFunctions.py:76)                                       */
  float epsilon;
} gccnmf_rt_config;
GCCNMF_API size_t gccnmf_rt_state_bytes(const gccnmf_rt_config* cfg);
/* W (F, K) f32; E (F, D) complex64 = expJOmegaTau (:248); windows (N) f32 (:186); H0 (K, 2) f32 seeded initial coefficients
 * (gccNMFFunctions.py:73 shape (K, 2)) or NULL when inference_iterations == 0.  Zeroes the rings and the history. */
GCCNMF_API int gccnmf_rt_init(gccnmf_handle* h, const gccnmf_rt_config* cfg, const float* W, const float* E,
                   const float* analysis_window, const float* synthesis_window, const float* H0, void* state,
                   size_t state_bytes, void* stream);
/* setTargetTDOARange (:272-276) and the attributes GCCNMFProcess sets (:136-151).  mode 0 boxcar / 1 window (:262-265).
 * localization_window >= 1 columns (GCCNMF_ERR_INVALID_ARGUMENT otherwise).  set_target = 0 keeps the device-resident target TDOA index (it is loop-carried when localisation is enabled). */
GCCNMF_API int gccnmf_rt_set_params(gccnmf_handle* h, const gccnmf_rt_config* cfg, void* state, size_t state_bytes,
                         float target_index, int set_target, float epsilon, float beta, float noise_floor, int mode,
                         int separation_enabled, int localization_enabled, int localization_window, void* stream);
/* processFrames: windowed (2, N, nT) f32 -> out (2, N, nT) f32 (device buffers); updates history / localisation.
 * forced_atom_mask: NULL, or a (K, nT) f64 atom mask that replaces the one derived from the per-atom TDOA argmax
 * (externally decided masks; teacher-forced parity tests). */
GCCNMF_API int gccnmf_rt_process_frames(gccnmf_handle* h, const gccnmf_rt_config* cfg, void* state, size_t state_bytes,
                             const float* windowed, float* out, const double* forced_atom_mask, void* stream);
/* One audio block through rings + processFrames (utils.py:99-116): in_block (2, B) f32 -> out_block (2, B) f32. */
GCCNMF_API int gccnmf_rt_process_block(gccnmf_handle* h, const gccnmf_rt_config* cfg, void* state, size_t state_bytes,
                            const float* in_block, float* out_block, const double* forced_atom_mask, void* stream);
/* The same block as an instantiated CUDA graph ([H2D of in_host ->] kernels [-> D2H to out_host]); in_host / out_host are
 * pinned HOST buffers or NULL; `stream` must be a capturable (non-default) stream.  *graph_exec receives a cudaGraphExec_t. */
GCCNMF_API int gccnmf_rt_graph_create(gccnmf_handle* h, const gccnmf_rt_config* cfg, void* state, size_t state_bytes,
                           float* in_block, float* out_block, const float* in_host, float* out_host, void** graph_exec,
                           void* stream);
GCCNMF_API int gccnmf_rt_graph_launch(gccnmf_handle* h, void* graph_exec, void* stream);
GCCNMF_API int gccnmf_rt_graph_destroy(gccnmf_handle* h, void* graph_exec);
/* Stream-ordered copy of one item of the block state to dst (device or pinned host memory): 0 gccPHAT (D, nT) f32,
 * 1 target TDOA index f32, 2 atom mask (K, nT) f64, 3 / 4 input / output spectrogram (2, F, nT) c64, 5 per-atom TDOA
 * argmax (K, nT) i32, 6 inferred H (K, 2 nT) f32, 7 GCC-PHAT history ring (D, history_length) f64, 8 its write index i32. */
GCCNMF_API int gccnmf_rt_export(gccnmf_handle* h, const gccnmf_rt_config* cfg, void* state, size_t state_bytes, int what,
                     void* dst, void* stream);

/* ---- the real-time block path for S independent streams (slots) in one state buffer ----------------------
 * The slots share the configuration, W, E, the windows and H0; each owns its rings, block counter, GCC-PHAT history, target
 * TDOA index and parameters, plus an `active` flag.  One block of every slot is the same five kernels (+ two per inference
 * iteration) as one stream, in one launch each, and one CUDA graph launch when captured.  Slot s computes bit for bit what a
 * single-stream state (gccnmf_rt_*, the S = 1 case of the same kernels) fed the same blocks and parameters computes.  An
 * inactive slot is skipped: its output slice is zeros, its input slice is ignored, its state stays as it was.  Buffers of all
 * slots are slot-major: in / out blocks (S, 2, B), windowed frames (S, 2, N, nT), forced atom masks (S, K, nT) f64.
 * Out-of-range num_streams (1 .. 4096), slot ranges and too small state buffers fail before anything is enqueued. */
typedef struct gccnmf_rtm_slot_params {
  float target_index; int set_target;      /* set_target = 0 keeps the device-resident target TDOA index             */
  float epsilon, beta, noise_floor;
  int mode;                                /* 0 boxcar, 1 window (:262-265)                                           */
  int separation_enabled, localization_enabled, localization_window;
  int active;                              /* 0: the slot is skipped by every block until re-activated                 */
} gccnmf_rtm_slot_params;
/* Host only; 0 for num_streams < 1 or an invalid configuration.  Grows linearly in num_streams. */
GCCNMF_API size_t gccnmf_rtm_state_bytes(const gccnmf_rt_config* cfg, int num_streams);
/* As gccnmf_rt_init, for every slot: all slots active, with the defaults of gccNMFProcessor.py:190-199. */
GCCNMF_API int gccnmf_rtm_init(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, const float* W, const float* E,
                    const float* analysis_window, const float* synthesis_window, const float* H0, void* state,
                    size_t state_bytes, void* stream);
/* Slots [first_slot, first_slot + count) go back to what gccnmf_rtm_init leaves (zeroed rings, history and counters, default
 * parameters, active); the other slots are untouched.  Stream-ordered: may sit between two launches of an instantiated graph. */
GCCNMF_API int gccnmf_rtm_reset_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state,
                           size_t state_bytes, int first_slot, int count, void* stream);
/* params: host array of `count` entries, consumed before the call returns. */
GCCNMF_API int gccnmf_rtm_set_params(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state,
                          size_t state_bytes, int first_slot, int count, const gccnmf_rtm_slot_params* params, void* stream);
GCCNMF_API int gccnmf_rtm_process_frames(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state,
                              size_t state_bytes, const float* windowed, float* out, const double* forced_atom_mask,
                              void* stream);
GCCNMF_API int gccnmf_rtm_process_block(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state,
                             size_t state_bytes, const float* in_blocks, float* out_blocks, const double* forced_atom_mask,
                             void* stream);
/* Launch / destroy with gccnmf_rt_graph_launch / gccnmf_rt_graph_destroy. */
GCCNMF_API int gccnmf_rtm_graph_create(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state,
                            size_t state_bytes, float* in_blocks, float* out_blocks, const float* in_host, float* out_host,
                            void** graph_exec, void* stream);
/* Item `what` of slot `slot`, as gccnmf_rt_export. */
GCCNMF_API int gccnmf_rtm_export(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state, size_t state_bytes,
                      int slot, int what, void* dst, void* stream);

/* ---- S streams, each separated into P sources: one output block per target TDOA (TARGET_MODE_MULTIPLE) ---------------
 * The multi-target rule of gccNMFFunctions.py:118-143 applied per block.  A slot has P target TDOA indexes tau_0 .. tau_{P-1}
 * in [0, D), 2 <= P <= 8.  For every atom k and frame t the winner is argmax_q gccNMF[tau_q][t][k] (the float32 values of the
 * per-atom contraction) under numpy.argmax's order: a NaN first, then the larger value, then the lower source index (so an
 * all-NaN column, which numpy.nanargmax rejects, and every tie go to the lowest source).  mask_q = (winner == q) (f64 0 / 1);
 * source q is then exactly the single-target filter and synthesis fed mask_q, overlap-added into its own output ring.  The P
 * masks partition the atoms, so the P outputs sum to the separation-off output up to float64 rounding of the mask sums.
 * Separation off: every source outputs the mixture.  Inactive slot: every source outputs zeros.
 * Targets: gccnmf_rtsep_set_targets, or with localisation on the P largest strict local maxima of the windowed GCC-PHAT mean in
 * ascending order (estimateTargetTDOAIndexesFromAngularSpectrum, gccNMFFunctions.py:94-116) become the targets of the NEXT
 * block; with fewer than P peaks the targets stay and status bit GCCNMF_RTSEP_STATUS_FEW_PEAKS is set (sticky until reset).
 * Defaults after init / reset_slots: tau_q = floor((2 q + 1) D / (2 P)).
 * Buffers: in blocks (S, 2, B), out blocks (S, P, 2, B), windowed frames in (S, 2, N, nT), out (S, P, 2, N, nT).
 * Export items 0 .. 8 as gccnmf_rt_export (2 and 4: source 0's), plus 9 targets (P) i32, 10 source masks (P, K, nT) f64,
 * 11 target values gccNMF[tau_q] (P, K, nT) f32, 12 output spectrograms (P, 2, F, nT) c64, 13 status word i32.
 * num_sources outside [2, 8], targets outside [0, D) and localisation with D < 3 fail before anything is enqueued. */
#define GCCNMF_RTSEP_MAX_SOURCES 8
#define GCCNMF_RTSEP_STATUS_FEW_PEAKS 1
/* Host only; 0 for an invalid configuration, num_streams or num_sources.  Grows linearly in num_streams. */
GCCNMF_API size_t gccnmf_rtsep_state_bytes(const gccnmf_rt_config* cfg, int num_streams, int num_sources);
GCCNMF_API int gccnmf_rtsep_init(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, const float* W,
                      const float* E, const float* analysis_window, const float* synthesis_window, const float* H0, void* state,
                      size_t state_bytes, void* stream);
GCCNMF_API int gccnmf_rtsep_reset_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state,
                             size_t state_bytes, int first_slot, int count, void* stream);
/* As gccnmf_rtm_set_params; mode, target_index and set_target are ignored. */
GCCNMF_API int gccnmf_rtsep_set_params(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state,
                            size_t state_bytes, int first_slot, int count, const gccnmf_rtm_slot_params* params, void* stream);
/* targets_host: count x P host array, consumed before the call returns; -1 keeps that source's target. */
GCCNMF_API int gccnmf_rtsep_set_targets(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state,
                             size_t state_bytes, int first_slot, int count, const int32_t* targets_host, void* stream);
GCCNMF_API int gccnmf_rtsep_process_frames(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state,
                                size_t state_bytes, const float* windowed, float* out, void* stream);
GCCNMF_API int gccnmf_rtsep_process_block(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state,
                               size_t state_bytes, const float* in_blocks, float* out_blocks, void* stream);
/* Launch / destroy with gccnmf_rt_graph_launch / gccnmf_rt_graph_destroy. */
GCCNMF_API int gccnmf_rtsep_graph_create(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state,
                              size_t state_bytes, float* in_blocks, float* out_blocks, const float* in_host, float* out_host,
                              void** graph_exec, void* stream);
GCCNMF_API int gccnmf_rtsep_export(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state,
                        size_t state_bytes, int slot, int what, void* dst, void* stream);

/* ---- S streams (x P sources) over a bank of dictionaries and steering tables ----------------------------------------------
 * The reference rebuilds a processor when its dictionary size / type or microphone spacing changes (gccNMFProcessor.py:131-157,
 * buildTheanoFunctions :238-270): a new W and expJOmegaTau, the same rings and GCC-PHAT history.  Here the state holds
 * num_dictionaries = Qd dictionary entries, entry i with its own K_i in [1, cfg.num_atoms = K_max] atoms, and num_steerings = Qe
 * steering entries (F, D), 1 <= Qd, Qe <= 64; every slot is on one entry of each.  N, hop, B, nT, D, the history length and the
 * inference settings stay engine-wide.  num_sources: 0 (one output per slot, as gccnmf_rtm_*) or 2 .. 8 (as gccnmf_rtsep_*).
 * Slot s on (i, j) computes bit for bit what a one-stream state built with (W_i, E_j) computes from the same blocks and
 * parameters: every output block and every export item.
 * - init: host arrays of Qd device pointers W_i (F, K_i) f32, Qd host ints K_i, Qd device pointers H0_i (K_i, 2) f32 (the array
 *   or its entries NULL when inference_iterations == 0) and Qe device pointers E_j (F, D) complex64.  Every slot on (0, 0).
 * - load_dictionary / load_steering rewrite one entry; assign moves slots [first_slot, first_slot + count) to the entries of
 *   the host arrays `dictionary` / `steering` (count each, -1 or a NULL array keeps the slot's entry).  All three are
 *   stream-ordered and may sit between two launches of an instantiated graph; they act from the next block on and keep the
 *   slot's rings, history, targets, block counter and parameters.  reset_slots also puts the slots back on (0, 0).
 * - Forced atom masks (num_sources = 0): (S, K_max, nT) f64; rows k >= K_i of a slot are ignored.
 * - export: items as gccnmf_rtm_export / gccnmf_rtsep_export, the K-shaped ones (2, 5, 6, 10, 11) at the K_i of the block
 *   they were computed in (of the slot's current dictionary before its first block; these wait for the stream to read K_i),
 *   plus 14: the slot's (dictionary, steering) entries (2) i32.
 * num_dictionaries = num_steerings = 0 in gccnmf_rtbank_state_bytes gives the gccnmf_rtm / gccnmf_rtsep size.  K_i outside
 * [1, K_max], entries outside the bank and more than 64 entries fail with GCCNMF_ERR_INVALID_ARGUMENT. */
#define GCCNMF_RTBANK_MAX_ENTRIES 64
#define GCCNMF_RTBANK_EXPORT_ASSIGNMENT 14
GCCNMF_API size_t gccnmf_rtbank_state_bytes(const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries,
                                 int num_steerings);
GCCNMF_API int gccnmf_rtbank_init(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries,
                       int num_steerings, void* state, size_t state_bytes, const float* const* W, const int* num_atoms,
                       const float* const* H0, const float* const* E, const float* analysis_window, const float* synthesis_window,
                       void* stream);
GCCNMF_API int gccnmf_rtbank_load_dictionary(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources,
                                  int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int index, const float* W,
                                  int num_atoms, const float* H0, void* stream);
GCCNMF_API int gccnmf_rtbank_load_steering(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources,
                                int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int index, const float* E,
                                void* stream);
GCCNMF_API int gccnmf_rtbank_assign(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries,
                         int num_steerings, void* state, size_t state_bytes, int first_slot, int count, const int32_t* dictionary,
                         const int32_t* steering, void* stream);
GCCNMF_API int gccnmf_rtbank_reset_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources,
                              int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int first_slot, int count,
                              void* stream);
/* As gccnmf_rtm_set_params (num_sources = 0) or gccnmf_rtsep_set_params. */
GCCNMF_API int gccnmf_rtbank_set_params(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources,
                             int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int first_slot, int count,
                             const gccnmf_rtm_slot_params* params, void* stream);
/* As gccnmf_rtsep_set_targets; needs num_sources >= 2. */
GCCNMF_API int gccnmf_rtbank_set_targets(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources,
                              int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int first_slot, int count,
                              const int32_t* targets_host, void* stream);
/* forced_atom_mask: NULL, or (S, K_max, nT) f64 with num_sources = 0. */
GCCNMF_API int gccnmf_rtbank_process_frames(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources,
                                 int num_dictionaries, int num_steerings, void* state, size_t state_bytes, const float* windowed,
                                 float* out, const double* forced_atom_mask, void* stream);
GCCNMF_API int gccnmf_rtbank_process_block(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources,
                                int num_dictionaries, int num_steerings, void* state, size_t state_bytes, const float* in_blocks,
                                float* out_blocks, const double* forced_atom_mask, void* stream);
/* Launch / destroy with gccnmf_rt_graph_launch / gccnmf_rt_graph_destroy. */
GCCNMF_API int gccnmf_rtbank_graph_create(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources,
                               int num_dictionaries, int num_steerings, void* state, size_t state_bytes, float* in_blocks,
                               float* out_blocks, const float* in_host, float* out_host, void** graph_exec, void* stream);
GCCNMF_API int gccnmf_rtbank_export(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources,
                         int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int slot, int what, void* dst,
                         void* stream);

/* ---- a11 streamed: the online / low-latency notebook loop for S streams ---------------------------------------------
 * onlineSpeechEnhancement.ipynb:406-447 / lowLatencySpeechEnhancement.ipynb:511-584 as performOnlineSpeechEnhancement computes
 * them in batch, one hop at a time.  Each call pushes hops * hop new samples per stream (1 <= hops <= hops_per_call) and emits
 * as many finished output samples per stream: output sample p is overlap-add sample p - L, L = Q hop - hop - z with
 * Q = ceil(N / hop) and z the first nonzero index of the synthesis weights w (N - hop - z when hop divides N; samples before the
 * first frame are zero).  Per frame: float64 rfft of
 * frame x analysis window rounded to complex64, PHAT coherence, angular spectrum, running maximum carried across calls, target =
 * argmax, all-TDOA GCC-NMF argmax per atom (tensor cores + float64 refinement, and a gated float64 launch when the refinement
 * list overflows), boxcar atom mask with the stream's epsilon, Wiener filter (W . mask) / rowsum(W) or, with inference, the
 * H-inferred filter, inverse FFT, then acc = float32(fma(w[r], frame[r], acc)) into an N-sample output ring in frame order and
 * gain x acc out.  One call is stream-ordered with no host synchronisation and can be captured as one CUDA graph.
 * Constraints: N a power of two in [32, 4096], 1 <= hop <= N, 1 <= C <= 64, D a power of two in [4, 128], 1 <= S <= 4096,
 * z <= (Q - 1) hop, and with inference (K + N / 2 + 1) x 4 <= 227 KiB. */
typedef struct gccnmf_ll_config {
  int window_size;           /* N                                                                       */
  int hop_size;              /* hop                                                                     */
  int hops_per_call;         /* C: the most hops one call may push                                      */
  int num_atoms;             /* K                                                                       */
  int num_tdoas;             /* D                                                                       */
  int num_streams;           /* S                                                                       */
  int inference_iterations;  /* 0: (W . mask) / rowsum(W); > 0: H-only KL updates of every frame from H0 */
  float sparsity_alpha;      /* of the inference updates (gccNMFFunctions.py:76)                        */
  float epsilon;
} gccnmf_ll_config;
/* Per-stream settings (host struct): epsilon of the boxcar atom mask (|argmax - target| < epsilon); active = 0 makes the
 * stream output zeros and leaves its state untouched; target_override >= 0 replaces the localised target TDOA index. */
typedef struct gccnmf_ll_stream_params {
  float epsilon;
  int active;
  int target_override;
} gccnmf_ll_stream_params;
/* 0 for an invalid configuration. */
GCCNMF_API size_t gccnmf_ll_state_bytes(const gccnmf_ll_config* cfg);
/* W (F, K) f32; E (F, D) complex128 expJOmegaTau; analysis_window (N) f64; synthesis_weights (N) f64 = w; gain g (applied to
 * every emitted sample); H0 (K, 2) f32 (NULL when inference_iterations == 0).  All five are DEVICE pointers.  init reads w back
 * on `stream` and waits for it (the latency depends on it), so it synchronises `stream` once; it fails before enqueueing
 * anything else when w starts too late.  Every stream starts empty and active, with epsilon 1 and no target override. */
GCCNMF_API int gccnmf_ll_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, const float* W, const double* E,
                   const double* analysis_window, const double* synthesis_weights, float gain, const float* H0, void* state,
                   size_t state_bytes, void* stream);
/* Streams [first, first + count) go back to an empty stream (rings zeroed, running maximum -inf, frame count 0); their
 * parameters stay. */
GCCNMF_API int gccnmf_ll_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int first,
                            int count, void* stream);
GCCNMF_API int gccnmf_ll_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int first,
                         int count, const gccnmf_ll_stream_params* params_host, void* stream);
/* in (S, 2, hops * hop) f32 -> out (S, 2, hops * hop) f32, device buffers. */
GCCNMF_API int gccnmf_ll_process(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int hops,
                      const float* in, float* out, void* stream);
/* gccnmf_ll_process(hops) as an instantiated CUDA graph ([H2D of in_host ->] kernels [-> D2H to out_host]); launch and destroy with
 * gccnmf_rt_graph_launch / gccnmf_rt_graph_destroy. */
GCCNMF_API int gccnmf_ll_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int hops,
                           float* in, float* out, const float* in_host, float* out_host, void** graph_exec, void* stream);
/* Items of the last call, which pushed `hops` hops (T = S hops columns, column s hops + i = frame i of stream s's call):
 *   0 X (2, F, T) c64   1 coherence (F, T) c64   2 angular (D, T) f64   3 accumulated max (D, T) f64   4 targets (T) i32
 *   5 TDOA argmax per atom (K, T) i32   6 atom masks (K, T) f32   7 Wiener filters (F, T) f32, or (2, F, T) with inference
 *   8 Y (2, F, T) c64   9 refined count (1) i32   10 status (1) i32: 1 when the float64 fallback ran   11 H (K, 2T) f32
 *   (inference only)   12 frame valid (T) i32: 0 for a frame that starts before the stream's first sample   13 carried
 *   accumulated max (S, D) f64 */
GCCNMF_API int gccnmf_ll_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int hops, int what,
                     void* dst, void* stream);

/* ---- a11 streamed, each stream separated into P sources: one output per target TDOA (TARGET_MODE_MULTIPLE) --------------
 * The multi-target rule of gccNMFFunctions.py:94-143 per frame of the gccnmf_ll_* loop.  A stream has P target TDOA indexes
 * tau_0 .. tau_{P-1} in [0, D), 2 <= P <= 8.  Per whole frame t of a call:
 * - targets: the running maximum is carried as in gccnmf_ll_*; the P largest strict local maxima of the frame's running maximum,
 *   ascending (estimateTargetTDOAIndexesFromAngularSpectrum), become the stream's targets.  With fewer than P peaks the targets
 *   stay and status bit GCCNMF_LLSEP_STATUS_FEW_PEAKS of the stream is set (sticky until reset).  After init / reset the
 *   targets are floor((2 q + 1) D / (2 P)).  A source's override (gccnmf_llsep_set_targets, >= 0) replaces its target.  Frames
 *   before the stream's first sample and inactive streams change nothing.
 * - values[q][k][t] = float32 of the float64 sum_f W[f][k] Re(coh[f][t] E[f][tau_q(t)]): the bits gccnmf_tdoa_gccnmf writes at
 *   (tau_q(t), k, t).  masks = gccnmf_coeff_mask of the values (numpy.nanargmax; ties go to the lower source); a (k, t) whose
 *   values are all NaN belongs to no source and sets bit GCCNMF_LLSEP_STATUS_ALL_NAN of the call's status.
 * - source q: the single-target Wiener filter with mask_q (with inference, on the H inferred once per frame and shared by the
 *   sources), inverse FFT, overlap-add into its own N-sample output ring and emit, at the latency and gain of gccnmf_ll_*.
 * Where no value is NaN the masks partition the atoms, so the P outputs add up to the output with every atom kept.  The epsilon
 * and target_override of gccnmf_ll_stream_params play no part; `active` does (an inactive stream outputs zeros).
 * Buffers: in (S, 2, hops hop), out (S, P, 2, hops hop).  Launch / destroy graphs with gccnmf_rt_graph_launch / _destroy.
 * Export: items 0 .. 3 and 11 .. 13 as gccnmf_ll_export, plus 14 column targets (T, P) i32, 15 values (P, K, T) f32, 16 masks
 * (P, K, T) f32, 17 Wiener filters (P, F, T) f32 or (P, 2, F, T) with inference, 18 Y (P, 2, F, T) c64, 19 stream status (S) i32,
 * 20 carried targets (S, P) i32, 21 the call's status (1) i32.  Items 4 .. 10 (the single-target chain) are refused.
 * num_sources outside [2, 8], overrides outside [0, D) other than -1, and T P or P K T (T = S hops_per_call) at or above 2^31
 * fail before anything is enqueued. */
#define GCCNMF_LLSEP_MAX_SOURCES 8
#define GCCNMF_LLSEP_STATUS_FEW_PEAKS 1
#define GCCNMF_LLSEP_STATUS_ALL_NAN 2
#define GCCNMF_LLSEP_EXPORT_TARGETS 14
#define GCCNMF_LLSEP_EXPORT_VALUES 15
#define GCCNMF_LLSEP_EXPORT_MASKS 16
#define GCCNMF_LLSEP_EXPORT_WIENER 17
#define GCCNMF_LLSEP_EXPORT_Y 18
#define GCCNMF_LLSEP_EXPORT_STREAM_STATUS 19
#define GCCNMF_LLSEP_EXPORT_CARRIED_TARGETS 20
#define GCCNMF_LLSEP_EXPORT_CALL_STATUS 21
/* Host only; 0 for an invalid configuration or num_sources.  Larger than gccnmf_ll_state_bytes of the same configuration. */
GCCNMF_API size_t gccnmf_llsep_state_bytes(const gccnmf_ll_config* cfg, int num_sources);
/* As gccnmf_ll_init; every stream also starts on the default targets with no overrides. */
GCCNMF_API int gccnmf_llsep_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, const float* W, const double* E,
                      const double* analysis_window, const double* synthesis_weights, float gain, const float* H0, void* state,
                      size_t state_bytes, void* stream);
/* As gccnmf_ll_reset_streams; targets back to the defaults and status cleared, overrides stay. */
GCCNMF_API int gccnmf_llsep_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes,
                               int first, int count, void* stream);
GCCNMF_API int gccnmf_llsep_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes,
                            int first, int count, const gccnmf_ll_stream_params* params_host, void* stream);
/* targets_host: count x P host array, consumed before the call returns; -1: the source follows the localisation. */
GCCNMF_API int gccnmf_llsep_set_targets(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes,
                             int first, int count, const int32_t* targets_host, void* stream);
GCCNMF_API int gccnmf_llsep_process(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes,
                         int hops, const float* in, float* out, void* stream);
GCCNMF_API int gccnmf_llsep_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes,
                              int hops, float* in, float* out, const float* in_host, float* out_host, void** graph_exec,
                              void* stream);
GCCNMF_API int gccnmf_llsep_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes,
                        int hops, int what, void* dst, void* stream);

/* ---- stream records: move a live stream to another stream index, engine, device or process -----------------------------------
 * A record is the persistent state of one stream (its counters and parameters, running maximum, input ring, output ring(s) and,
 * with sources, its targets, overrides and status) behind a header.  It does not depend on num_streams, hops_per_call, the
 * stream index or the device.  A stream saved after a call and loaded anywhere compatible produces, from the next call on, the
 * bytes it would have produced had it never moved.  Compatible: the same gccnmf_ll_config fields other than num_streams and
 * hops_per_call (compared bit for bit), the same num_sources, the same synthesis weights and gain.
 * These entries are the low-latency engine's, one family for both of its forms (num_sources 0 for gccnmf_ll_*, 2 .. 8 for
 * gccnmf_llsep_*).
 * Records live in a caller-owned HOST buffer (pinned for asynchronous copies): `count` records of gccnmf_llrec_record_bytes
 * each, record i for stream first + i.  `workspace` is device staging of gccnmf_llrec_workspace_bytes(count) bytes, at least
 * 4-byte aligned (16-byte aligned for the fast copy).
 * save: reads the engine's synthesis weights and gain back on `stream` and waits for them (their digest goes into the header),
 *   then one copy kernel into the staging and one device-to-host copy; the host buffer is complete when `stream` reaches it.
 *   The streams are not changed (reset or deactivate them afterwards if they are to stop here).
 * load: checks magic, ABI version, kind, num_sources, payload size and configuration of every record on the host, without
 *   touching the device.  Only when all of them match does it read the synthesis weights and gain back (one wait on `stream`)
 *   to check the digest.  Then one host-to-device copy and one copy kernel; the streams' state is replaced from the next call on.
 *   Other streams, the graphs and the shared state are untouched.  A refused record enqueues no kernel and no host-to-device
 *   copy. */
#define GCCNMF_RECORD_MAGIC 0x52534347u   /* "GCSR" */
#define GCCNMF_RECORD_KIND_LL 2
#define GCCNMF_RECORD_HEADER_BYTES 256    /* the payload starts here in every record */
typedef struct gccnmf_record_header {
  uint32_t magic;
  int32_t abi_version;                    /* GCCNMF_ABI_VERSION of the library that wrote it */
  int32_t kind;
  int32_t num_sources;                    /* 0: gccnmf_ll_* */
  uint64_t payload_bytes;
  uint64_t synthesis_digest;              /* FNV-1a 64 of the synthesis weights' bytes followed by the gain's */
  int32_t config[16];                     /* the config struct's fields in order (num_streams and hops_per_call 0), then 0 */
} gccnmf_record_header;
/* num_sources: 0 for a gccnmf_ll_* engine, else the gccnmf_llsep_* engine's.  Host only; 0 for an invalid configuration or
 * num_sources, or count < 1. */
GCCNMF_API size_t gccnmf_llrec_record_bytes(const gccnmf_ll_config* cfg, int num_sources);
GCCNMF_API size_t gccnmf_llrec_workspace_bytes(const gccnmf_ll_config* cfg, int num_sources, int count);
GCCNMF_API int gccnmf_llrec_save_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes,
                              int first, int count, void* record, size_t record_bytes, void* workspace, size_t workspace_bytes,
                              void* stream);
GCCNMF_API int gccnmf_llrec_load_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes,
                              int first, int count, const void* record, size_t record_bytes, void* workspace,
                              size_t workspace_bytes, void* stream);

/* ---- localisation over a sliding window of each stream's recent frames ----------------------------------------------------------
 * The low-latency engine of gccnmf_ll_* (num_sources 0) or gccnmf_llsep_* (2 .. 8) with a history of history_length = Lh frames per
 * stream, 0 <= Lh <= 1024.  Every entry takes (num_sources, history_length) after the config and does what its gccnmf_ll_* /
 * gccnmf_llsep_* namesake does; with Lh = 0 the engine, its state size, its launches and its records are those of the namesakes.
 * - History ring: every whole frame of an active stream writes its angular spectrum column (export item 2, float64) into the
 *   stream's (D, Lh) ring at the write index, which then moves on (mod Lh).  The running maximum and its carry advance as before,
 *   whatever the window.  Frames before the first sample and inactive streams change nothing.  init and reset zero the ring and
 *   set the write index and the window to 0.
 * - Window w per stream, 0 <= w <= Lh (gccnmf_llhist_set_window; from the next call, and allowed between launches of a graph):
 *   w = 0 keeps the running-maximum rule of the namesakes.  w >= 1: per frame, mean[d] = the nanmean of the newest w ring columns,
 *   summed in float64 newest first, skipping NaN (NaN when all are NaN); the zero columns of a ring that has seen fewer than w
 *   frames count in the denominator.  This is rt_localize's rule (gccnmf_rt_*).  The target is then the argmax of the mean
 *   (numpy.argmax's order; target_override still wins), or with sources the P largest strict local maxima of the mean with the
 *   hold rule, status bit and overrides of gccnmf_llsep_*.  After w frames without NaN, an earlier NaN no longer matters.
 * - Export: the namesakes' items plus 22 the rings (S, D, Lh) f64, 23 the write indexes (S) i32, 24 the windows (S) i32 and 25 the
 *   call's window means (D, T) f64 (NaN for the streams with w = 0).  Items 22 .. 25 need Lh > 0.
 * - Records (gccnmf_llhist_record_bytes / workspace_bytes / save_streams / load_streams): gccnmf_llrec_*'s, with the ring, its
 *   write index and the window after the other regions, and Lh in config[9] of the header; a load requires an equal Lh.  With
 *   Lh = 0 the records are byte-identical to gccnmf_llrec_*'s, and each family loads the other's.
 * Lh outside [0, 1024], a window outside [0, Lh], items 22 .. 25 or set_window with Lh = 0, set_targets with num_sources 0, and
 * S D Lh at or above 2^31 fail before anything is enqueued. */
#define GCCNMF_LLHIST_MAX_HISTORY 1024
#define GCCNMF_LLHIST_EXPORT_RING 22
#define GCCNMF_LLHIST_EXPORT_INDEX 23
#define GCCNMF_LLHIST_EXPORT_WINDOWS 24
#define GCCNMF_LLHIST_EXPORT_MEANS 25
/* Host only; 0 for an invalid configuration, num_sources or history_length. */
GCCNMF_API size_t gccnmf_llhist_state_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length);
GCCNMF_API int gccnmf_llhist_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, const float* W,
                       const double* E, const double* analysis_window, const double* synthesis_weights, float gain, const float* H0,
                       void* state, size_t state_bytes, void* stream);
/* Also zeroes the streams' rings and sets their write index and window to 0. */
GCCNMF_API int gccnmf_llhist_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                                size_t state_bytes, int first, int count, void* stream);
GCCNMF_API int gccnmf_llhist_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                             size_t state_bytes, int first, int count, const gccnmf_ll_stream_params* params_host, void* stream);
/* num_sources >= 2 only. */
GCCNMF_API int gccnmf_llhist_set_targets(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                              size_t state_bytes, int first, int count, const int32_t* targets_host, void* stream);
/* windows_host: count host int32, consumed before the call returns, each in [0, history_length]. */
GCCNMF_API int gccnmf_llhist_set_window(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                             size_t state_bytes, int first, int count, const int32_t* windows_host, void* stream);
GCCNMF_API int gccnmf_llhist_process(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                          size_t state_bytes, int hops, const float* in, float* out, void* stream);
GCCNMF_API int gccnmf_llhist_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                               size_t state_bytes, int hops, float* in, float* out, const float* in_host, float* out_host,
                               void** graph_exec, void* stream);
GCCNMF_API int gccnmf_llhist_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                         size_t state_bytes, int hops, int what, void* dst, void* stream);
GCCNMF_API size_t gccnmf_llhist_record_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length);
GCCNMF_API size_t gccnmf_llhist_workspace_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int count);
GCCNMF_API int gccnmf_llhist_save_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                               size_t state_bytes, int first, int count, void* record, size_t record_bytes, void* workspace,
                               size_t workspace_bytes, void* stream);
GCCNMF_API int gccnmf_llhist_load_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                               size_t state_bytes, int first, int count, const void* record, size_t record_bytes, void* workspace,
                               size_t workspace_bytes, void* stream);

/* ---- a bank of steering tables: each stream on its own microphone spacing ------------------------------------------------------
 * The engine of gccnmf_llhist_* (num_sources 0 or 2 .. 8, history_length 0 .. 1024) with num_steerings = Qe steering tables,
 * 0 <= Qe <= 64.  Every entry takes (num_sources, history_length, num_steerings) after the config and does what its gccnmf_llhist_*
 * namesake does; with Qe = 0 the engine, its state size, its launches and its records are the namesake's.
 * - Tables: init takes E_0 .. E_{Qe-1} as one device array (Qe, F, D) complex128, each as gccnmf_ll_init takes E.  Stream s is on
 *   entry assign[s]; init and reset_streams put it on entry 0.  N, hop, D, K, W, H0, the windows, the synthesis, P and Lh are the
 *   engine's.  A stream on entry j computes, bit for bit, every sample and export item a gccnmf_llhist_* engine with the same
 *   num_sources and history_length built with E_j computes from the same input and settings.
 * - load_steering (table j <- a device (F, D) complex128 array) and assign (streams -> entries) act from the next call, may sit between
 *   launches of a graph, and keep every other part of the streams: rings, running maximum, history, window, targets, overrides, hop
 *   count and parameters.  Those are indexed by TDOA, so a new table changes only the columns computed from then on.
 * - Export: the namesake's items plus 26 the assignment (S) i32 (Qe >= 1).
 * - Records (record_bytes / workspace_bytes / save_streams / load_streams): with Qe = 0 gccnmf_llhist_*'s.  With Qe >= 1 the kind is
 *   GCCNMF_RECORD_KIND_LLBANK and the header a gccnmf_llbank_record_header: gccnmf_record_header's fields, then the content digests
 *   (GCCNMF_RTREC_DIGEST_*, computed on the device) of the dictionary (W (F, K) f32, then H0 (K, 2) f32 with inference) and of the
 *   stream's steering table as stored ((F, D) complex128).  A load checks every host field first (refused: nothing enqueued), then
 *   the synthesis digest and the destination's digests (one wait on `stream` each); it refuses, with the state unchanged, a record
 *   whose dictionary differs or whose table no entry holds, and otherwise puts the stream on the LOWEST entry with that table.  The
 *   workspace must be 8-byte aligned.  Records do not move between bank and non-bank engines.
 * Qe outside [0, 64], an entry outside [0, Qe), item 26 with Qe = 0 and the namesake's refusals fail before anything is enqueued. */
#define GCCNMF_LLBANK_MAX_STEERINGS 64
#define GCCNMF_LLBANK_EXPORT_ASSIGNMENT 26
#define GCCNMF_RECORD_KIND_LLBANK 3
typedef struct gccnmf_llbank_record_header {
  uint32_t magic;                         /* the fields up to config are those of gccnmf_record_header */
  int32_t abi_version;
  int32_t kind;                           /* GCCNMF_RECORD_KIND_LLBANK */
  int32_t num_sources;
  uint64_t payload_bytes;
  uint64_t synthesis_digest;
  int32_t config[16];
  uint64_t dictionary_digest;
  uint64_t steering_digest;               /* of the table the stream was on */
} gccnmf_llbank_record_header;
/* Host only; 0 for an invalid configuration, num_sources, history_length or num_steerings. */
GCCNMF_API size_t gccnmf_llbank_state_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings);
GCCNMF_API int gccnmf_llbank_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings,
                       const float* W, const double* E, const double* analysis_window, const double* synthesis_weights, float gain,
                       const float* H0, void* state, size_t state_bytes, void* stream);
/* E: one (F, D) complex128 DEVICE table for entry `entry`. */
GCCNMF_API int gccnmf_llbank_load_steering(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                                int num_steerings, void* state, size_t state_bytes, int entry, const double* E, void* stream);
/* entries_host: count host int32 in [0, num_steerings), consumed before the call returns. */
GCCNMF_API int gccnmf_llbank_assign(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings,
                         void* state, size_t state_bytes, int first, int count, const int32_t* entries_host, void* stream);
GCCNMF_API int gccnmf_llbank_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                                int num_steerings, void* state, size_t state_bytes, int first, int count, void* stream);
GCCNMF_API int gccnmf_llbank_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings,
                             void* state, size_t state_bytes, int first, int count, const gccnmf_ll_stream_params* params_host,
                             void* stream);
GCCNMF_API int gccnmf_llbank_set_targets(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                              int num_steerings, void* state, size_t state_bytes, int first, int count, const int32_t* targets_host,
                              void* stream);
GCCNMF_API int gccnmf_llbank_set_window(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings,
                             void* state, size_t state_bytes, int first, int count, const int32_t* windows_host, void* stream);
GCCNMF_API int gccnmf_llbank_process(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings,
                          void* state, size_t state_bytes, int hops, const float* in, float* out, void* stream);
GCCNMF_API int gccnmf_llbank_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                               int num_steerings, void* state, size_t state_bytes, int hops, float* in, float* out,
                               const float* in_host, float* out_host, void** graph_exec, void* stream);
GCCNMF_API int gccnmf_llbank_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings,
                         void* state, size_t state_bytes, int hops, int what, void* dst, void* stream);
GCCNMF_API size_t gccnmf_llbank_record_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings);
GCCNMF_API size_t gccnmf_llbank_workspace_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings,
                                     int count);
GCCNMF_API int gccnmf_llbank_save_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                               int num_steerings, void* state, size_t state_bytes, int first, int count, void* record,
                               size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream);
GCCNMF_API int gccnmf_llbank_load_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                               int num_steerings, void* state, size_t state_bytes, int first, int count, const void* record,
                               size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream);

/* ---- a bank of dictionaries: each stream on its own dictionary and steering table ------------------------------------------------
 * The engine of gccnmf_llbank_* with num_dictionaries = Qd dictionaries, 1 <= Qd <= 64, and 1 <= Qe <= 64 steering tables.  Every
 * entry takes (num_sources, history_length, num_dictionaries, num_steerings) after the config.  cfg.num_atoms is Kmax, the most
 * atoms an entry may hold.  Stream s is on dictionary entry dictionary[s] and steering entry steering[s]; init and reset_streams put it
 * on (0, 0).  A stream on dictionary i (W_i with K_i atoms) and table j computes, bit for bit, every sample and export item (rows
 * < K_i of the K-shaped ones) a gccnmf_llhist_* engine with the same num_sources and history_length built with (W_i, E_j) computes.
 * - init takes W as Qd DEVICE pointers to (F, K_i) f32, num_atoms as Qd host K_i in [1, Kmax] and, with inference, H0 as Qd device
 *   pointers to (K_i, 2) f32; E as gccnmf_llbank_init takes it.  load_dictionary(index, W, num_atoms, H0) replaces one entry.
 * - assign(first, count, dictionary_host, steering_host): -1 (or a NULL array) keeps a stream's entry.  assign and both load_* calls
 *   are stream-ordered, act from the next call, may sit between launches of a graph and keep every other part of the streams.
 * - Export: the llbank items plus 27 the dictionary assignment (S) i32 and 28 the K_i table (Qd) i32.  K-shaped items keep Kmax rows;
 *   rows >= K_i of a column are argmax -1 and masks, values, source masks and H 0.
 * - Records: GCCNMF_RECORD_KIND_LLBANK with a gccnmf_llbank_record_header whose config.num_atoms is the stream's K_i and whose
 *   dictionary digest is that of W_i (F, K_i) (then H0_i (K_i, 2) with inference): the record a gccnmf_llbank_* engine built with W_i
 *   writes, so records move both ways between the two families.  A load puts the stream on the lowest entries holding its dictionary
 *   (same digest and K) and its table, and refuses, with the state unchanged, a dictionary no entry holds or a K mismatch.
 * K_i outside [1, Kmax], an entry outside the bank, Qd or Qe outside [1, 64], (Kmax + F) x 4 bytes over 227 KB with inference and the
 * llbank refusals fail before anything is enqueued. */
#define GCCNMF_LLDICT_MAX_DICTIONARIES 64
#define GCCNMF_LLDICT_EXPORT_DICTIONARY_ASSIGNMENT 27
#define GCCNMF_LLDICT_EXPORT_DICTIONARY_ATOMS 28
/* Host only; 0 for an invalid configuration or argument. */
GCCNMF_API size_t gccnmf_lldict_state_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                                 int num_steerings);
GCCNMF_API int gccnmf_lldict_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                       int num_steerings, const float* const* W, const int* num_atoms, const float* const* H0, const double* E,
                       const double* analysis_window, const double* synthesis_weights, float gain, void* state, size_t state_bytes,
                       void* stream);
GCCNMF_API int gccnmf_lldict_load_dictionary(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                                  int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int index, const float* W,
                                  int num_atoms, const float* H0, void* stream);
GCCNMF_API int gccnmf_lldict_load_steering(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                                int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int index, const double* E,
                                void* stream);
GCCNMF_API int gccnmf_lldict_assign(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                         int num_steerings, void* state, size_t state_bytes, int first, int count, const int32_t* dictionary_host,
                         const int32_t* steering_host, void* stream);
GCCNMF_API int gccnmf_lldict_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                                int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int first, int count, void* stream);
GCCNMF_API int gccnmf_lldict_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                             int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int first, int count,
                             const gccnmf_ll_stream_params* params_host, void* stream);
GCCNMF_API int gccnmf_lldict_set_targets(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                              int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int first, int count,
                              const int32_t* targets_host, void* stream);
GCCNMF_API int gccnmf_lldict_set_window(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                             int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int first, int count,
                             const int32_t* windows_host, void* stream);
GCCNMF_API int gccnmf_lldict_process(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                          int num_steerings, void* state, size_t state_bytes, int hops, const float* in, float* out, void* stream);
GCCNMF_API int gccnmf_lldict_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                               int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int hops, float* in, float* out,
                               const float* in_host, float* out_host, void** graph_exec, void* stream);
GCCNMF_API int gccnmf_lldict_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                         int num_steerings, void* state, size_t state_bytes, int hops, int what, void* dst, void* stream);
GCCNMF_API size_t gccnmf_lldict_record_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                                  int num_steerings);
GCCNMF_API size_t gccnmf_lldict_workspace_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                                     int num_steerings, int count);
GCCNMF_API int gccnmf_lldict_save_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                               int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int first, int count, void* record,
                               size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream);
GCCNMF_API int gccnmf_lldict_load_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length,
                               int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int first, int count,
                               const void* record, size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream);

/* ---- real-time stream records: move a live slot to another slot, engine, engine form, device or process ---------------------
 * One family for every real-time form, with the arguments of gccnmf_rtbank_*: (num_streams, num_sources, num_dictionaries,
 * num_steerings) = (1, 0, 0, 0) for gccnmf_rt_*, (S, 0, 0, 0) for gccnmf_rtm_*, (S, P, 0, 0) for gccnmf_rtsep_* and
 * (S, P, Qd, Qe) for a bank.  A record is the persistent state of one slot (its parameters, block counter, history index and
 * target, GCC-PHAT history, input ring, output ring(s) and, with sources, its targets and status) behind a gccnmf_rtrec_header.
 * It does not depend on num_streams, the slot index, num_dictionaries, num_steerings, num_atoms (K_max) or the device.  A slot
 * saved between blocks and loaded into a compatible slot computes, from the next block on, the bytes it would have computed had
 * it never moved.  Compatible: the same gccnmf_rt_config fields other than num_atoms (compared bit for bit), the same
 * num_sources, the same windows, and a dictionary entry and a steering entry whose content digests equal the record's.  The
 * record names its entries by content, not by index: a load puts the slot on the LOWEST destination entry of each kind whose
 * digest (and, for a dictionary, K_i) matches, and writes that into the slot's bank assignment.  The empty bank (rt, rtm,
 * rtsep) counts as one dictionary of num_atoms atoms and one steering table.
 * Content digest (GCCNMF_RTREC_DIGEST_*): the input is a sequence of n 32-bit words cut into chunks of 1024 words; chunk j gets
 * c_j = FNV-1a 64 over its words (h = (h ^ w) * 0x100000001b3 from 0xcbf29ce484222325); the digest is FNV-1a 64 over the words
 * (n_lo, n_hi, c_0 lo, c_0 hi, c_1 lo, ...).  It is applied to the windows (analysis then synthesis, 2 N f32), to dictionary
 * entry i (W_i (F, K_i) f32, then H0_i (K_i, 2) f32 when inference_iterations > 0) and to steering entry j (its stored E^T,
 * (D, Fp) complex64 with Fp = (F + 3) & ~3, the bins F .. Fp - 1 zero).
 * Records live in a caller-owned HOST buffer (pinned for asynchronous copies): `count` records of gccnmf_rtrec_record_bytes
 * each, record i for slot first + i.  `workspace` is device memory of gccnmf_rtrec_workspace_bytes(count) bytes, 16-byte aligned.
 * save: the digest kernels, one copy kernel that writes `count` whole records (header included) into the workspace, one
 *   device-to-host copy; no host wait.  The slots are not changed.
 * load: checks magic, ABI version, kind, num_sources, payload size and configuration of every record on the host (refused: nothing
 *   enqueued).  Then the digest kernels on the destination, one read-back of the digests and K_i (one wait on `stream`), and the
 *   mapping of every record's entries (refused: only those read-only kernels ran).  Then one host-to-device copy of the records,
 *   one copy kernel (which also writes the bank assignment) and, with a bank, the sort of the slots by dictionary.  Other slots,
 *   the graphs and the shared region are untouched; both entries are stream-ordered and may sit between two graph launches.
 *   K-shaped exports between a load and the next block still describe the destination slot's last block. */
#define GCCNMF_RECORD_KIND_RT 1
#define GCCNMF_RTREC_DIGEST_CHUNK_WORDS 1024
#define GCCNMF_RTREC_DIGEST_BASIS 0xcbf29ce484222325ull
#define GCCNMF_RTREC_DIGEST_PRIME 0x100000001b3ull
typedef struct gccnmf_rtrec_header {
  uint32_t magic;                         /* the first 24 bytes are those of gccnmf_record_header */
  int32_t abi_version;
  int32_t kind;                           /* GCCNMF_RECORD_KIND_RT */
  int32_t num_sources;                    /* 0 or 2 .. 8 */
  uint64_t payload_bytes;
  uint64_t windows_digest;
  uint64_t dictionary_digest;             /* of the dictionary entry the slot was on */
  uint64_t steering_digest;               /* of the steering entry the slot was on */
  int32_t dictionary_atoms;               /* that entry's K_i */
  int32_t reserved;                       /* 0 */
  int32_t config[16];                     /* the config struct's fields in order (num_atoms 0), then 0 */
} gccnmf_rtrec_header;
/* Host only; 0 for an invalid configuration, num_sources or bank, or count < 1. */
GCCNMF_API size_t gccnmf_rtrec_record_bytes(const gccnmf_rt_config* cfg, int num_sources);
GCCNMF_API size_t gccnmf_rtrec_workspace_bytes(const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries,
                                    int num_steerings, int count);
GCCNMF_API int gccnmf_rtrec_save_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources,
                            int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int first, int count,
                            void* record, size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream);
GCCNMF_API int gccnmf_rtrec_load_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources,
                            int num_dictionaries, int num_steerings, void* state, size_t state_bytes, int first, int count,
                            const void* record, size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream);

/*
 * The building block the KL-NMF loop runs on (klnmf_tma.cu): the same 3-product contraction, TMA-fed, over operands
 * that are pre-split into bf16 hi/lo planes and kept in ONE orientation each; an operand contracted over its
 * non-contiguous dimension is consumed MN-major.  Test / diagnostics entry: splits the float32 operands into planes
 * in the workspace, then DT (N, M) row-major = (A . B^T)^T.
 *   a_mn_major = 0: A is (M, Kc) row-major;  1: A is (Kc, M) row-major.   b_mn_major likewise with N.
 *   tile_n in {112, 128, 176, 208, 240, 256}, and 104 / 120 with a K-major B (dual-N tiles);  splits > 1: `splits` partial slabs
 *   DT[z] over k ranges (N * M floats each).
 *   timing: device uint64[8 x CTAs] stamps (layout: gccnmf_debug_timing) or NULL.
 */
/* Tile plan of the KL-NMF loop on a device with sm_count SMs (host logic only; callable without a GPU):
 * out[0] tile width of the W.H contractions, out[1] of the H update, out[2] / out[3] tile width / k-splits of the W-update
 * numerator, out[4] n tiles of the H update, out[5..7] CTAs of the three launches.  < 0: shape not covered by this path. */
GCCNMF_API int gccnmf_klnmf_tile_plan(int sm_count, int F, int T2, int K, int* out);
GCCNMF_API size_t gccnmf_gemm_planes_workspace_bytes(int M, int N, int Kc);
/* Diagnostics: while `stamps` (device uint64) is non-NULL every plane GEMM launched through the handle appends 8 values
 * per CTA at a running offset: [0] / [7] %globaltimer ns at CTA start / end, [1..6] clock64 at start, first stage full,
 * last MMA issued, producer done, accumulator complete, epilogue end.  Returns the offset reached; reset != 0 rewinds. */
GCCNMF_API int64_t gccnmf_debug_timing(gccnmf_handle* h, unsigned long long* stamps, int reset);
GCCNMF_API int gccnmf_gemm_planes(gccnmf_handle* h, const float* A, int a_mn_major, const float* B, int b_mn_major, float* DT,
                       int M, int N, int Kc, int tile_n, int splits, void* workspace, size_t workspace_bytes,
                       unsigned long long* timing, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GCCNMF_B200_H_ */
