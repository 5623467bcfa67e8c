/*
 * posediff_b200.h -- C ABI of the H100-native PoseDiffusion sampling hot path.
 *
 * The reference (facebookresearch/PoseDiffusion) is pure Python + PyTorch ATen; it has NO C ABI,
 * plugin or FFI layer (SURVEY.md §8b).  This header therefore declares the entry points a
 * reference-side binding (ctypes, see INTEGRATION.md) needs in order to replace, one for one, the
 * Python call sites of the hot path:
 *
 *   pdb_denoiser_load      <- load_state_dict of `diffuser.model.*`      (pose_diffusion/demo.py:56-57,
 *                                                                          models/pose_diffusion_model.py:57-61)
 *   pdb_denoiser_forward   <- Denoiser.forward(x, t, z)                  (models/denoiser.py:53-76)
 *   pdb_p_sample           <- GaussianDiffusion.p_sample                 (models/gaussian_diffuser.py:249-282)
 *   pdb_matches_pack       <- matches_dict -> device tensors, pair_idx   (util/geometry_guided_sampling.py:16-45,
 *                                                                          util/match_extraction.py:50-77 output format)
 *   pdb_matches_pack_colmap<- colmap_keypoint_to_pytorch3d fused into the packer (util/match_extraction.py:50-77)
 *   pdb_sampson_eval       <- compute_sampson_distance + backward        (util/geometry_guided_sampling.py:129-172)
 *   pdb_ggs                <- geometry_guided_sampling (5 x GGS_optimize) (util/geometry_guided_sampling.py:14-126)
 *   pdb_sample_loop        <- GaussianDiffusion.sample / p_sample_loop   (models/gaussian_diffuser.py:285-306)
 *   pdb_sample_loop_ddim   <- the fewer-step sampling the reference's `sampling_timesteps` names but never built (:79, :150-154,
 *                             :303-306): a DDIM prefix in k < 100 steps, then the same guided DDPM + GGS tail
 *   pdb_sample_loop_ddim_guided <- the same with the guided tail in g' < g DDIM jumps, GGS after each (no reference
 *                             counterpart: the reference's guided steps are always the g DDPM steps)
 *   pdb_sample_loop_host   <- the same call with HOST buffers (demo.py:108 as a user sees it: features and
 *                             matches on the host, poses back on the host)
 *   pdb_sample_loop_host_matches <- the same call starting from the reference's matches_dict arrays (demo.py:94-108:
 *                             extract_match output straight into the sampler); packing overlaps the unguided steps
 *   pdb_sample_loop_host_matches_ddim <- that call on the loop of pdb_sample_loop_ddim_guided
 *   pdb_images_preprocess_host <- load_and_preprocess_images after PIL decoding (util/load_img_folder.py: float conversion,
 *                             centre crop, bilinear resize; demo.py:51, test.py:172)
 *
 * Conventions: plain pointers and sizes only (no torch types).  `*_dev` pointers are CUDA device pointers
 * on the context's device, `*_host` are host pointers, `stream` is a cudaStream_t passed as void*
 * (NULL = legacy default stream).  All floating point data is IEEE fp32 unless stated; pose layout is the
 * reference's "absT_quaR_logFL" encoding [B, N, 9] = (T xyz, quaternion wxyz, log focal xy), row-major.
 * Every function returns PDB_OK (0) or a negative pdb_status; pdb_last_error() gives the message.
 * There is no CPU fallback: every compute entry point fails with PDB_ERR_CUDA if no sm_90 device exists.
 */
#ifndef POSEDIFF_B200_H
#define POSEDIFF_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PDB_ABI_VERSION 2

typedef enum pdb_status {
  PDB_OK = 0,
  PDB_ERR_INVALID = -1,   /* bad argument (mirrors the reference's ValueError / NotImplementedError sites) */
  PDB_ERR_CUDA = -2,      /* CUDA runtime failure, or no Hopper (sm_90) device */
  PDB_ERR_STATE = -3,     /* e.g. weights not loaded */
  PDB_ERR_LIMIT = -4      /* size beyond a compiled limit (frames > PDB_MAX_FRAMES, ...) */
} pdb_status;

#define PDB_TARGET_DIM 9       /* models/denoiser.py:26 */
#define PDB_Z_DIM 384          /* DINO ViT-S/16 CLS width, models/denoiser.py:28 */
#define PDB_NUM_TIMESTEPS 100  /* models/gaussian_diffuser.py:78 */
#define PDB_MAX_FRAMES 128     /* frames per sequence supported by the kernels */
#define PDB_NUM_WEIGHT_TENSORS 108
#define PDB_GGS_PHASES 5       /* util/geometry_guided_sampling.py:47-64 */

typedef struct pdb_context pdb_context; /* one per (process, GPU) */
typedef struct pdb_matches pdb_matches; /* device-resident packed correspondences of ONE sequence */

/* cfgs/default.yaml:6-13 -> kwargs of GGS_optimize (util/geometry_guided_sampling.py:74-81). */
typedef struct pdb_ggs_config {
  double alpha;         /* 1e-4 */
  double learning_rate; /* 1e-2 */
  int32_t iter_num;     /* 100 (doubled for the all-parameter phases, :86-87) */
  double sampson_max;   /* 10 */
  double min_matches;   /* 10; <= 0 disables the early exit (:103) */
  double momentum;      /* 0.9 (hard-coded in the reference, :89) */
} pdb_ggs_config;

/* What the reference prints per phase ("t=.. | sampson=..", :124) plus the early-exit notice (:107). */
typedef struct pdb_ggs_stats {
  float sampson[PDB_GGS_PHASES];    /* mean(min(err, sampson_max)) of the last evaluated iteration */
  int32_t iters[PDB_GGS_PHASES];    /* SGD updates actually applied in the phase */
  int32_t dropped[PDB_GGS_PHASES];  /* 1 if the phase stopped on "insufficient valid matches" */
  int32_t n_valid[PDB_GGS_PHASES];  /* valid matches at the last evaluated iteration */
} pdb_ggs_stats;

/* ---- context ---------------------------------------------------------------------------------- */
int pdb_abi_version(void);
int pdb_create(pdb_context** out, int device_ordinal);
void pdb_destroy(pdb_context* ctx);
const char* pdb_last_error(const pdb_context* ctx); /* ctx may be NULL: last creation error */
int pdb_device_info(const pdb_context* ctx, int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor);
/* number of kernels this library has launched since creation (bench.py's gpu_launches) */
int64_t pdb_launch_count(const pdb_context* ctx);

/* Kernel timing for bench.py's roofline line: when enabled, every GGS / denoiser launch is bracketed by CUDA
 * events on its own stream; pdb_profile_read synchronises those events and returns the summed device time (ms)
 * and launch counts since the last read. */
int pdb_profile_enable(pdb_context* ctx, int32_t on);
int pdb_profile_read(pdb_context* ctx, double* ggs_ms, int64_t* ggs_launches, double* denoiser_ms, int64_t* denoiser_launches);

/* Debug probe (not part of the reference surface): per-CTA cycle sums of a persistent kernel's stages.  enable = 1: the GGS kernel
 * of single-sequence calls, out[cta][8] = {stage3 norms, stage1, stage2b, exchange, stage2a, iterations, next stage 0, stage3 update};
 * enable = 2: the fp32 denoiser kernel, out[cta][8] = {barrier, tile load + LayerNorm, linear item, attention, tail, steps, -, -};
 * enable = 0 frees the buffer. */
int pdb_debug_ggs_clocks(pdb_context* ctx, int32_t enable, int64_t* out, int32_t max_ctas);

/* Swap-AB tensor-core tiles (weights on the 128-row M side, 32 / 64 / 96 tokens on the N side) for GEMMs with at most 96 tokens
 * and O % 128 == 0; default off (without split-K only O/128 CTAs stream the weights).  Debug / measurement switch. */
int pdb_debug_tc_swap(pdb_context* ctx, int32_t on);

/* Stage hand-over inside the persistent fp32 denoiser kernel: 0 (default) = plain floats and a group barrier per stage; 1 = every
 * activation travels as a 64-bit {fp32, version tag} word and consumers poll the data itself, no barrier between the 43 stages of
 * a diffusion step.  Same arithmetic, bit-identical results; the flagged variant is slower (every CTA polling
 * the 80 KB flagged tiles loads L2).  Debug / measurement switch (environment: PDB_DEN_FLAG). */
int pdb_debug_denoiser_handover(pdb_context* ctx, int32_t flagged);

/* Reproducible mode.  on = 1: every sampling entry (pdb_ggs, pdb_sample_loop*, pdb_p_sample, pdb_denoiser_forward) returns the
 * same bits on every call with the same inputs (weights, z, draws, match sets, GGS config) on the same library build and GPU
 * model, whatever else runs on the GPU: GGS runs a kernel whose floating-point sums all have a fixed order and exchanges its
 * partial gradients through the flag-carrying slots (no one-hop reductions), and the tensor-core GEMMs run without split-K.
 * on = 0 (the default): the faster kernels, whose floating-point sums depend on scheduling.  Affects only work enqueued after the
 * call; the debug outputs (pdb_debug_ggs_clocks, pdb_sampson_eval) are outside the contract.  Any other value: PDB_ERR_INVALID,
 * the mode unchanged. */
int pdb_set_reproducible(pdb_context* ctx, int on);

/* Denoiser engine: 0 = auto (exact-fp32 persistent kernel below 128 tokens per GPU, wgmma/TMA tensor-core tiles with TF32
 * products at or above), 1 = always fp32, 2 = always tensor cores. */
int pdb_denoiser_engine(pdb_context* ctx, int32_t mode);

/* Test entry of the tensor-core linear layer (wgmma tf32 fed by TMA; csrc/tc_linear.cuh):
 * Y[S,O] = relu?(X[S,K] @ W[O,K]^T + bias + residual); K % 32 == 0, O % 64 == 0, fp32 in / out, TF32 products. */
int pdb_debug_tc_linear(pdb_context* ctx, const float* x_dev, const float* w_dev, const float* bias_dev,
                        const float* residual_dev, float* y_dev, int32_t S, int32_t O, int32_t K, int32_t relu,
                        void* stream);

/* DDPM schedule exactly as GaussianDiffusion.init_diff_hyper builds it (models/gaussian_diffuser.py:136-187;
 * "custom" = float64 linspace(beta_1, beta_T, 100), cumprod, cast to float32).  HOST-ONLY helper, needs no GPU:
 * out[100][8] = {sqrt_recip_alphas_cumprod, sqrt_recipm1_alphas_cumprod, posterior_mean_coef1,
 * posterior_mean_coef2, exp(0.5*posterior_log_variance_clipped), posterior_log_variance_clipped, betas,
 * alphas_cumprod}. */
int pdb_schedule_table(float* out, double beta_1, double beta_T);

/* DDIM step table (Song et al. 2021, eq. 12) for `steps` denoiser evaluations of which the last `guide_below` (g) are guided:
 * the unguided prefix takes k = steps - g strided steps, 1 <= k <= 100 - g, tau_j = (g - 1) + floor(j * (100 - g) / k), entry i
 * jumping tau_{k-i} -> tau_{k-i-1} (the last lands on x_{g-1}, or on x0 when g = 0).  HOST-ONLY, float64 arithmetic cast to float32:
 * t_out[steps] = the timestep each entry evaluates the network at; coef_out[steps][8]: prefix entries {a_t, b_t, c1, c2, sigma, s,
 * abar_t, abar_s} with x' = c1 * (a_t x - b_t eps) + c2 x + sigma * noise, sigma = eta sqrt((1-abar_s)/(1-abar_t)) sqrt(1 -
 * abar_t/abar_s), c2 = sqrt(1 - abar_s - sigma^2) / sqrt(1 - abar_t), c1 = sqrt(abar_s) - c2 sqrt(abar_t), abar_{-1} = 1; entries
 * k .. steps-1 are the pdb_schedule_table rows of timesteps g-1 .. 0 (the guided tail stays DDPM).  With k = 100 - g and eta = 1
 * the prefix rows equal the DDPM posterior rows up to rounding.  PDB_ERR_INVALID for k out of range, eta < 0 or not finite, or
 * an eta > 1 large enough to make 1 - abar_s - sigma^2 negative.  It is pdb_ddim_table_guided with guided_steps = guide_below. */
int pdb_ddim_table(int32_t steps, int32_t guide_below, double eta, double beta_1, double beta_T, int32_t* t_out, float* coef_out);

/* pdb_ddim_table with the guided tail in g' = `guided_steps` denoiser evaluations, 1 <= g' <= g (g' = 0 when g = 0): the prefix
 * takes k = steps - g' steps (still 1 <= k <= 100 - g).  With g' == g entries k .. steps-1 are the DDPM rows, exactly as
 * pdb_ddim_table writes them; with g' < g they are g' DDIM jumps of the same form and eta as the prefix's, entry k + i jumping
 * tau'_{g'-i} -> tau'_{g'-i-1}, tau'_j = floor(j * g / g') - 1 (tau'_{g'} = g - 1, tau'_0 = -1 = x0).  The samplers add no noise
 * on guided jumps (sigma is tabulated all the same).  HOST-ONLY; PDB_ERR_INVALID as pdb_ddim_table, and for g' out of range. */
int pdb_ddim_table_guided(int32_t steps, int32_t guide_below, int32_t guided_steps, double eta, double beta_1, double beta_T,
                          int32_t* t_out, float* coef_out);

/* ---- denoiser weights ---------------------------------------------------------------------------
 * `tensors[i]` (host or device, fp32, contiguous) in the order of the reference state_dict below
 * `diffuser.model.`:  time_embed.linear.0.{weight,bias}, time_embed.linear.2.{weight,bias},
 * _first.{weight[512,702],bias}, then for layer 0..7: self_attn.in_proj_{weight,bias},
 * self_attn.out_proj.{weight,bias}, linear1.{weight,bias}, linear2.{weight,bias}, norm1.{weight,bias},
 * norm2.{weight,bias}; then _last.0.{weight,bias}, _last.1.{weight,bias}, _last.3.{weight,bias}.
 * The library re-lays them out for the kernels and tabulates the timestep-embedding MLP for t in [0,100). */
int pdb_denoiser_load(pdb_context* ctx, const float* const* tensors, int32_t count, void* stream);

/* eps[B,N,9] = Denoiser(x[B,N,9], t, z[B,N,384]); one integer timestep for the whole batch, as the
 * sampler uses it (gaussian_diffuser.py:265). */
int pdb_denoiser_forward(pdb_context* ctx, const float* x_dev, int32_t t, const float* z_dev, int32_t batch,
                         int32_t frames, float* eps_dev, void* stream);

/* One ancestral step WITHOUT guidance (gaussian_diffuser.py:249-282): writes x0 (may be NULL), the posterior
 * mean (may be NULL) and pred = mean + sigma_t * noise (noise_dev NULL or t == 0 -> pred = mean). */
int pdb_p_sample(pdb_context* ctx, const float* x_dev, int32_t t, const float* z_dev, const float* noise_dev,
                 int32_t batch, int32_t frames, float* pred_dev, float* mean_dev, float* x0_dev, void* stream);

/* ---- correspondences ----------------------------------------------------------------------------
 * Input is the reference's matches_dict (demo.py:82-87): kp1/kp2 float64 [m,2] pixel coordinates,
 * i12 int64 [m,2] frame indices, img_shape (frames, 3, height, width).  Rows with equal (i12[0], i12[1])
 * are expected in contiguous runs (any run order; a pair may recur).  Packed ONCE into device-resident
 * fp32 (u1,v1,u2,v2) quads, pair-segmented and padded to 32-row rounds; pair/segment indexing is exact.
 * `on_device` != 0 means the three arrays are device pointers. */
int pdb_matches_pack(pdb_context* ctx, const double* kp1, const double* kp2, const int64_t* i12, int64_t m_total,
                     int32_t frames, int32_t height, int32_t width, int32_t on_device, void* stream,
                     pdb_matches** out);
/* The same ingestion from the COLMAP / hloc tables, fusing the reference's remap (util/match_extraction.py:50-77):
 * keypoints[i] = [kp_counts[i], 2] COLMAP pixel coordinates of image i (float32 or float64, `kp_is_f64`),
 * pair_ids[p] = (r, q) 1-based image ids, pair_matches[p] = [match_counts[p], 2] keypoint index pairs (NULL or count 0 = no
 * matches), bboxes_xyxy [n_images, 4] and scales [n_images] from load_and_preprocess_images.  kp' = (kp - 0.5 - bbox_xy) * scale. */
int pdb_matches_pack_colmap(pdb_context* ctx, int32_t n_images, const void* const* keypoints, const int32_t* kp_counts,
                            int32_t kp_is_f64, int32_t n_pairs, const int32_t* pair_ids, const int32_t* const* pair_matches,
                            const int32_t* match_counts, const double* bboxes_xyxy, const double* scales, int32_t frames,
                            int32_t height, int32_t width, void* stream, pdb_matches** out);
void pdb_matches_free(pdb_matches* m);
int pdb_matches_info(const pdb_matches* m, int64_t* m_total, int32_t* segments, int64_t* rounds, int32_t* frames);

/* Layout of the packed match stream in HBM for match sets packed on this context from now on (csrc/ggs_layout.cuh):
 * 1 = paired (the default: segments padded to 64-row units, the two matches of a lane component-interleaved so that the
 * 128-bit loads are directly the operand pairs of the packed fp32x2 pipe), 0 = plain (one float4 per match, segments padded
 * to 32-row rounds; the layout the round-1 numbers were measured with).  Same 16 B per match, same results (tests/
 * test_gpu_layout.py); the environment variable PDB_GGS_LAYOUT=plain|paired overrides the default at pdb_create. */
int pdb_ggs_layout(pdb_context* ctx, int32_t layout);
int pdb_ggs_layout_get(const pdb_context* ctx); /* the layout new match sets are packed in (0 / 1) */

/* Host-only layout probe (no GPU, no context; test infrastructure): writes the stream image pdb_matches_pack would upload
 * for reference-format matches -- segs_out [*nseg][4] = {first_round, count, frame_a, frame_b}, pts_out [*rounds * 32 * 4]
 * floats.  With segs_out or pts_out NULL it only reports *nseg and *rounds.  PDB_ERR_LIMIT if the buffers are too small. */
int pdb_debug_pack_layout(const double* kp1, const double* kp2, const int64_t* i12, int64_t m_total, int32_t frames,
                          int32_t layout, int32_t* segs_out, int32_t max_segs, float* pts_out, int64_t max_rounds,
                          int32_t* nseg, int64_t* rounds);

/* compute_sampson_distance + backward for one sequence: grad_dev[N,9] = d mean(valid err) / d pose,
 * scalars_dev[4] = {loss, n_valid, logged (= mean(min(err, max)) over all matches), 0}.  Optional per-segment
 * dumps: F_dev[segments,9] (F' = F^T), G_dev[segments,9] (sum over valid matches of d err / d F').
 * update flags as in GGS_optimize (:71-73). */
int pdb_sampson_eval(pdb_context* ctx, const pdb_matches* m, const float* pose_dev, int32_t update_R,
                     int32_t update_T, int32_t update_FL, double sampson_max, float* grad_dev, float* scalars_dev,
                     float* F_dev, float* G_dev, void* stream);

/* geometry_guided_sampling for `batch` independent sequences: pose_dev[batch, N, 9] is optimised in place.
 * stats_dev (device, may be NULL) receives `batch` pdb_ggs_stats records, without any host synchronisation. */
int pdb_ggs(pdb_context* ctx, pdb_matches* const* problems, int32_t batch, float* pose_dev,
            const pdb_ggs_config* cfg, pdb_ggs_stats* stats_dev, void* stream);

/* ---- sampler ------------------------------------------------------------------------------------
 * p_sample_loop: draws_dev[T+1, B, N, 9] holds the Gaussian draws in the reference's order (draws[0] = x_T,
 * draws[1+k] = noise of loop iteration k, i.e. t = T-1-k; unused on guided steps and at t = 0).
 * problems == NULL -> no guidance; otherwise problems[n_problems] holds ONE match set per sequence: n_problems must equal
 * `batch` and every set must have been packed for `frames` frames (PDB_ERR_INVALID otherwise -- the kernels index
 * problems[b] and stride the pose by the set's frame count).  cond_start_step as in p_sample (:270).  trail_dev may be NULL, else
 * [T+1, B, N, 9].  stats_dev may be NULL, else [cond_start_step, batch] records (row 0 = first guided step).
 * Every sampling-loop entry point refuses its arguments before anything is enqueued: NULL pointers, batch or frames < 1,
 * frames > PDB_MAX_FRAMES (PDB_ERR_LIMIT), no weights loaded (PDB_ERR_STATE), match sets without cfg or as above, cfg->iter_num
 * < 0, and the DDIM entries' step-table refusals.  Only a match set that fails to pack in pdb_sample_loop_host_matches* is
 * found later, while the unguided steps run. */
int pdb_sample_loop(pdb_context* ctx, const float* z_dev, const float* draws_dev, int32_t batch, int32_t frames,
                    pdb_matches* const* problems, int32_t n_problems, const pdb_ggs_config* cfg,
                    int32_t cond_start_step, float* pose_dev, float* trail_dev, pdb_ggs_stats* stats_dev, void* stream);

/* pdb_sample_loop with a DDIM prefix: `steps` denoiser evaluations in all, of which g = clamp(cond_start_step, 0, 100) are the
 * guided tail (exactly pdb_sample_loop's guided DDPM steps + GGS; problems / cfg / stats as there) and k = steps - g the unguided
 * prefix on the pdb_ddim_table schedule.  draws_dev [1 + k, B, N, 9] when eta > 0 (draws[0] = x_T, draws[1 + i] = noise of
 * prefix step i), [1, B, N, 9] when eta == 0 (x_T only).  trail_dev may be NULL, else [1 + steps, B, N, 9].  problems == NULL
 * with cond_start_step > 0 runs the prefix alone and leaves x_{g-1} in pose_dev (a caller's own guidance takes over from there).
 * PDB_ERR_INVALID before anything is enqueued for k out of range, a bad eta or a NULL draws pointer; PDB_ERR_LIMIT for frames >
 * PDB_MAX_FRAMES.  The step table is copied (stream-ordered) into a buffer the context owns; concurrent loops on one context
 * must share a stream.  It is pdb_sample_loop_ddim_guided with guided_steps = g. */
int pdb_sample_loop_ddim(pdb_context* ctx, const float* z_dev, const float* draws_dev, int32_t batch, int32_t frames, int32_t steps,
                         double eta, pdb_matches* const* problems, int32_t n_problems, const pdb_ggs_config* cfg,
                         int32_t cond_start_step, float* pose_dev, float* trail_dev, pdb_ggs_stats* stats_dev, void* stream);

/* pdb_sample_loop_ddim with the guided tail in g' = `guided_steps` jumps (pdb_ddim_table_guided): k = steps - g' prefix steps,
 * then per jump one denoiser step to the DDIM mean (no noise, no draw) and GGS on it in place, with the same cfg (its iteration
 * counts are not rescaled by the stride).  g' == g is exactly pdb_sample_loop_ddim.  trail_dev [1 + k + g', B, N, 9], stats_dev
 * [g', batch] records.  PDB_ERR_INVALID before anything is enqueued for g' outside [1, g] (0 when g = 0), k outside [1, 100 - g]
 * or a bad eta. */
int pdb_sample_loop_ddim_guided(pdb_context* ctx, const float* z_dev, const float* draws_dev, int32_t batch, int32_t frames,
                                int32_t steps, double eta, int32_t guided_steps, pdb_matches* const* problems, int32_t n_problems,
                                const pdb_ggs_config* cfg, int32_t cond_start_step, float* pose_dev, float* trail_dev,
                                pdb_ggs_stats* stats_dev, void* stream);

/* The same with host buffers (pinned or pageable): copies z and the draws in, runs, copies pose (and the
 * optional trajectory / stats) out, synchronises the stream.  This is the end-to-end call bench.py times. */
int pdb_sample_loop_host(pdb_context* ctx, const float* z_host, const float* draws_host, int32_t batch,
                         int32_t frames, pdb_matches* const* problems, int32_t n_problems, const pdb_ggs_config* cfg,
                         int32_t cond_start_step, float* pose_host, float* trail_host, pdb_ggs_stats* stats_host,
                         void* stream);

/* The end-to-end call that starts from the reference's match format: kp1[b] / kp2[b] (float64 [m_total[b], 2]) and i12[b]
 * (int64 [m_total[b], 2]) are the HOST arrays of sequence b's matches_dict (util/match_extraction.py:50-77), as pdb_matches_pack
 * takes them.  The sets are packed and uploaded while the unguided steps t = T-1 .. cond_start_step already run on the GPU, then
 * the guided steps follow; the packed sets are released before the call returns.  Results are those of pdb_matches_pack +
 * pdb_sample_loop_host.  cfg must not be NULL.  A set that fails to pack (e.g. an i12 index outside the frames) is refused
 * while the unguided steps run: the stream is then synchronised and the sets packed so far are released. */
int pdb_sample_loop_host_matches(pdb_context* ctx, const float* z_host, const float* draws_host, int32_t batch, int32_t frames,
                                 const double* const* kp1, const double* const* kp2, const int64_t* const* i12,
                                 const int64_t* m_total, int32_t height, int32_t width, const pdb_ggs_config* cfg,
                                 int32_t cond_start_step, float* pose_host, float* trail_host, pdb_ggs_stats* stats_host,
                                 void* stream);

/* pdb_sample_loop_host_matches on the loop of pdb_sample_loop_ddim_guided: the sets are packed while the DDIM prefix runs.
 * draws_host [1 + k, B, N, 9] for eta > 0, [1, B, N, 9] for eta == 0; trail_host [1 + k + g', B, N, 9]; stats_host [g', batch].
 * The same refusals as pdb_sample_loop_ddim_guided, before anything is enqueued; a set that fails to pack as in
 * pdb_sample_loop_host_matches. */
int pdb_sample_loop_host_matches_ddim(pdb_context* ctx, const float* z_host, const float* draws_host, int32_t batch, int32_t frames,
                                      int32_t steps, double eta, int32_t guided_steps, const double* const* kp1,
                                      const double* const* kp2, const int64_t* const* i12, const int64_t* m_total, int32_t height,
                                      int32_t width, const pdb_ggs_config* cfg, int32_t cond_start_step, float* pose_host,
                                      float* trail_host, pdb_ggs_stats* stats_host, void* stream);

/* ---- image features (widened row, SURVEY 8f-2) ---------------------------------------------------
 * z = MultiScaleImageFeatureExtractor(image) (models/image_feature_extractor.py:27-87): the DINO ViT-S/16 backbone that the
 * reference pulls from torch.hub ("facebookresearch/dino:main", dino_vits16 -- third-party, restated in oracle/dino_vit.py),
 * applied to the ResNet-normalised image at each scale factor (bilinear resize, align_corners=False), class-token features
 * averaged over the scales (:74-83).  Projections run as wgmma/TMA tiles with TF32 products (fp32 accumulate).
 *
 * `tensors[i]` (fp32, contiguous) in the hub checkpoint's state_dict order (`image_feature_extractor._net.*`): cls_token,
 * pos_embed[1,197,384], patch_embed.proj.{weight[384,3,16,16],bias}, then for block 0..11: norm1.{weight,bias},
 * attn.qkv.{weight[1152,384],bias}, attn.proj.{weight,bias}, norm2.{weight,bias}, mlp.fc1.{weight[1536,384],bias},
 * mlp.fc2.{weight[384,1536],bias}; then norm.{weight,bias}.  numels[i] is checked against that layout. */
#define PDB_VIT_NUM_TENSORS 150
int pdb_vit_load(pdb_context* ctx, const float* const* tensors, const int64_t* numels, int32_t count, int32_t on_device,
                 void* stream);
/* interpolate_pos_encoding of the hub model for a grid_h x grid_w patch grid: bicubic resampling of the 14x14 table with the
 * scale factor (grid + 0.1) / 14 (torch F.interpolate semantics, align_corners=False).  HOST-ONLY helper, needs no GPU:
 * pos_embed_host [197,384] -> out_host [1 + grid_h*grid_w, 384].  (14, 14) means a square input and returns the stored table;
 * the hub model resamples a 14x14 grid of a non-square image (e.g. 224x232), which pdb_extract_features does too. */
int pdb_vit_pos_table(const float* pos_embed_host, int32_t grid_h, int32_t grid_w, float* out_host);
/* images_dev [n,3,H,W] in [0,1] (what load_and_preprocess_images / the dataloader produce) -> z_dev [n,384].
 * scale_factors as in cfgs/default.yaml (1, 1/2, 1/3); empty -> PDB_ERR_INVALID (the reference raises ValueError, :75-76).
 * PDB_ERR_LIMIT, before any kernel is launched, for more than 4 scales, more than 256 tokens per image at a scale, or more
 * than 65535 images.
 * tokens_debug_dev (may be NULL): receives the residual stream [sum over scales of n*(1+gh*gw), 384] (scale-major, image, token)
 * after stage `debug_stage` (0 = prepare_tokens, k = block k) -- the parity tests' probe. */
int pdb_extract_features(pdb_context* ctx, const float* images_dev, int32_t n_images, int32_t height, int32_t width,
                         const double* scale_factors, int32_t n_scales, float* z_dev, float* tokens_debug_dev,
                         int32_t debug_stage, void* stream);
/* The same with host buffers: copies the images in, z out, synchronises the stream. */
int pdb_extract_features_host(pdb_context* ctx, const float* images_host, int32_t n_images, int32_t height, int32_t width,
                              const double* scale_factors, int32_t n_scales, float* z_host, void* stream);

/* ---- image preprocessing ----------------------------------------------------------------------------
 * load_and_preprocess_images (util/load_img_folder.py) after decoding: frame i is rgb_host[i], HOST uint8 HWC of
 * hw[i] = {H, W} with row pitch 3*W (frames may differ in size); crop[i] = {top, left, side} is its square crop.
 * images_dev [n,3,out_size,out_size] receives crop / 255 (IEEE division) resized bilinearly (align_corners=False, no antialias;
 * ATen's CPU index and weight arithmetic, so a crop with side == out_size is copied exactly).  Only the crop columns of the rows
 * the resize reads are uploaded.  Synchronises the stream before returning, so the frames may be freed afterwards.
 * PDB_ERR_INVALID for n <= 0, out_size <= 0, a NULL pointer, or a crop outside its image or with side < 2. */
int pdb_images_preprocess_host(pdb_context* ctx, int32_t n, const uint8_t* const* rgb_host, const int32_t* hw,
                               const int32_t* crop, int32_t out_size, float* images_dev, void* stream);

/* ---- post-loop geometry (widened row, SURVEY 8f-3) -----------------------------------------------
 * pose_encoding_to_camera for "absT_quaR_logFL" (util/camera_transform.py:64-105): pose_dev [count,9] -> R_dev [count,3,3]
 * (pytorch3d quaternion_to_matrix, real part first, two_s = 2/|q|^2), T_dev [count,3], focal_dev [count,2] =
 * clamp(exp(pose[7:9] + log_focal_length_bias), min_focal_length, max_focal_length) (defaults 1.8, 0.1, 20). */
int pdb_pose_to_camera(pdb_context* ctx, const float* pose_dev, int32_t count, double log_focal_length_bias,
                       double min_focal_length, double max_focal_length, float* R_dev, float* T_dev, float* focal_dev,
                       void* stream);
/* camera_to_rel_deg (util/metric.py:14-48): R/T of `batch` sequences of `frames` cameras ([batch*frames,3,3], [batch*frames,3],
 * pytorch3d row-vector convention) -> r_deg_dev / t_deg_dev [batch * frames*(frames-1)/2]: relative rotation / translation
 * direction error in degrees for every pair i < j (torch.combinations order, sequence major).  invalid_dev[0] becomes non-zero
 * where the reference would raise ValueError (relative-rotation trace outside [-1-1e-4, 3+1e-4]). */
int pdb_rel_pose_error(pdb_context* ctx, const float* R_pred_dev, const float* T_pred_dev, const float* R_gt_dev,
                       const float* T_gt_dev, int32_t batch, int32_t frames, float* r_deg_dev, float* t_deg_dev,
                       int32_t* invalid_dev, void* stream);

/* 7-dof ("Umeyama") alignment of predicted cameras to target cameras before the absolute rotation error
 * (demo.py:126-128: pytorch3d.ops.corresponding_cameras_alignment(cameras_src, cameras_tgt, estimate_scale=True,
 * mode="extrinsics", eps=1e-9); third-party algorithm restated in csrc/align.cuh).  R [count,3,3], T [count,3] in pytorch3d's
 * row-vector convention; R_out / T_out = the aligned source cameras, align_dev[13] = {align_R (9), align_T (3), scale}. */
int pdb_cameras_align(pdb_context* ctx, const float* R_src_dev, const float* T_src_dev, const float* R_tgt_dev,
                      const float* T_tgt_dev, int32_t count, int32_t estimate_scale, double eps, float* R_out_dev,
                      float* T_out_dev, float* align_dev, void* stream);

/* ---- training (GaussianDiffusion.p_losses + Denoiser, models/gaussian_diffuser.py:308-341) -----------------------------------
 * params[108] are the denoiser parameters in pdb_denoiser_load order, device fp32, contiguous, 16-byte aligned; they are read
 * directly on every call (only `_first.weight`, whose 702-float rows TMA cannot address, is copied into the workspace padded to
 * 704 columns).  The workspace (pdb_train_workspace_bytes, device, 16-byte aligned) is owned by the caller: the forward writes
 * the activations the backward needs into it, the backward also uses it as scratch.  At most 64 frames per sequence.
 * Dropout: element e of site s (0 attention weights, 1 after out-proj, 2 after ReLU, 3 after linear2) of layer l is kept when
 * Philox4x32-10(key = seed, counter = {e >> 2, e >> 34, l << 8 | s, 0}) word e & 3 >= floor(p * 2^32); kept values are scaled by
 * 1 / (1 - p).  Elements are numbered row-major over [batch, heads, frames, frames] (site 0) and [batch * frames, width]. */
int64_t pdb_train_workspace_bytes(int32_t batch, int32_t frames); /* 0 for an unsupported shape */
/* x_start, noise [B,N,9]; t_dev [B] int32 in [0,100); z [B,N,384]; loss_type 0 = l1, 1 = l2.  Writes x_t = q_sample(x_start, t, noise),
 * loss [B,N,9] (reduction none, against the noise) and x0 = predict_start_from_noise(x_t, t, eps).  The caller validates t: a value
 * outside [0,100) is clamped where the kernels index the schedule (no out-of-bounds read), its outputs are meaningless, and
 * pdb_train_backward on that workspace fails with PDB_ERR_INVALID. */
int pdb_train_forward(pdb_context* ctx, const float* const* params, const float* x_start_dev, const int32_t* t_dev, const float* noise_dev,
                      const float* z_dev, int32_t batch, int32_t frames, float dropout_p, uint64_t seed, int32_t loss_type, void* workspace,
                      float* loss_dev, float* x_t_dev, float* x0_dev, void* stream);
/* grads[108] (device, parameter shapes) are overwritten with d(sum(grad_loss * loss) + sum(grad_x0 * x0)) / d params; grad_loss or
 * grad_x0 may be NULL (zero).  Synchronises the stream once to read the workspace header (shape, loss type, dropout seed, the
 * timestep flag).  Bit-reproducible: no floating-point atomics. */
int pdb_train_backward(pdb_context* ctx, const float* const* params, void* workspace, const float* grad_loss_dev, const float* grad_x0_dev,
                       float* const* grads, void* stream);
/* pdb_train_backward that also writes grad_z_dev [B,N,384] = d(...) / d z (NULL: exactly pdb_train_backward).  The 108 parameter
 * gradients do not depend on whether grad_z_dev is given. */
int pdb_train_backward_z(pdb_context* ctx, const float* const* params, void* workspace, const float* grad_loss_dev, const float* grad_x0_dev,
                         float* const* grads, float* grad_z_dev, void* stream);
/* Denoiser.forward with a backward (models/denoiser.py:53-76 under autograd): the same engine, workspace size and dropout rule as
 * the p_losses pair above.  eps_dev [B,N,9] = Denoiser(x_dev [B,N,9], t_dev[b] (int32 [B], one timestep per sequence), z_dev
 * [B,N,384]) with the activations saved in the workspace.  Timesteps outside [0,100) are handled as in pdb_train_forward.  The
 * workspace header records which forward filled it: pdb_train_backward[_z] refuses a pdb_denoiser_grad_forward workspace with
 * PDB_ERR_STATE, and pdb_denoiser_grad_backward a pdb_train_forward one. */
int pdb_denoiser_grad_forward(pdb_context* ctx, const float* const* params, const float* x_dev, const int32_t* t_dev, const float* z_dev,
                              int32_t batch, int32_t frames, float dropout_p, uint64_t seed, void* workspace, float* eps_dev, void* stream);
/* From grad_eps_dev [B,N,9] = dL/deps: grads[108] are overwritten with dL/d params (grads NULL: no parameter gradient, and only the
 * input-gradient chain runs: no weight, bias, _first or time-MLP gradient kernel), grad_x_dev [B,N,9] with dL/dx (through the
 * harmonic embedding and the raw pose columns of _first), grad_z_dev [B,N,384] with dL/dz; either may be NULL, but not all three.
 * Synchronises the stream once to read the workspace header.  Bit-reproducible: no floating-point atomics. */
int pdb_denoiser_grad_backward(pdb_context* ctx, const float* const* params, void* workspace, const float* grad_eps_dev,
                               float* const* grads, float* grad_x_dev, float* grad_z_dev, void* stream);
/* camera_to_pose_encoding, "absT_quaR_logFL" (util/camera_transform.py:108-129): R [count,3,3], T [count,3], focal [count,2] ->
 * pose [count,9] = T | matrix_to_quaternion(R) with the real part made non-negative | log(clamp(focal, min, max)) - bias. */
int pdb_camera_to_pose(pdb_context* ctx, const float* R_dev, const float* T_dev, const float* focal_dev, int32_t count,
                       double log_focal_length_bias, double min_focal_length, double max_focal_length, float* pose_dev, void* stream);
/* HOST-ONLY: out[i] = 1 if element offset + i of (layer, site) is kept under the dropout rule above, else 0. */
int pdb_dropout_mask_host(uint64_t seed, int32_t layer, int32_t site, int64_t offset, int64_t count, float dropout_p, uint8_t* out);

/* ---- training the image backbone (MultiScaleImageFeatureExtractor with freeze=False) --------------------------------------------
 * tensors[150] are the DINO ViT-S/16 parameters in pdb_vit_load order, device fp32, contiguous, 16-byte aligned, read where they
 * are on every call (pdb_vit_load is not needed and its copy is not used).  LayerNorm is applied explicitly (not folded into the
 * qkv / fc1 weights as pdb_extract_features does), so z differs from pdb_extract_features' z by the folding's rounding.
 * The workspace (device, 16-byte aligned, pdb_vit_train_workspace_bytes) is owned by the caller: the forward saves the activations
 * the backward needs in it, the backward also uses it as scratch.  Same shape limits as pdb_extract_features. */
int64_t pdb_vit_train_workspace_bytes(int32_t n_images, int32_t height, int32_t width, const double* scale_factors,
                                      int32_t n_scales); /* 0 for an unsupported shape */
/* images_dev [n,3,H,W] in [0,1] -> z_dev [n,384].  Synchronises the stream once per resampled scale (position-table taps upload). */
int pdb_vit_train_forward(pdb_context* ctx, const float* const* tensors, const float* images_dev, int32_t n_images, int32_t height,
                          int32_t width, const double* scale_factors, int32_t n_scales, void* workspace, float* z_dev, void* stream);
/* grads[150] (device, parameter shapes) are overwritten with d(sum(grad_z * z)) / d tensors; there is no gradient to the images.
 * Synchronises the stream once to read the workspace header.  Bit-reproducible: no floating-point atomics. */
int pdb_vit_backward(pdb_context* ctx, const float* const* tensors, void* workspace, const float* grad_z_dev, float* const* grads,
                     void* stream);

#ifdef __cplusplus
}
#endif
#endif /* POSEDIFF_B200_H */
