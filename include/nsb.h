/* nsb.h -- C ABI of libnsb.so: the H100-native (sm_90a) NeRSemble render hot path.
 *
 * Plain C: raw DEVICE pointers, sizes, scalar hparams, an explicit cudaStream_t (passed as
 * void*).  No C++/torch types.  Every entry point returns 0 on success, non-zero on error;
 * nsb_last_error() returns a thread-local message.  The library allocates nothing that
 * outlives a call (caller provides outputs and workspaces) and keeps no global mutable state
 * besides the error string, so it is re-entrant across streams (the reference trainer and
 * its viewer thread can render concurrently: engine/nersemble_trainer.py:38-40).
 *
 * Each entry point replaces a third-party call of the reference (paths relative to
 * /root/reference/src/nersemble/):
 *
 *   nsb_field_forward      tcnn.Encoding x8 + stack/rearrange/window/einsum + tcnn mlp_base/mlp_head
 *                          + nerfstudio MLP x8 + se3_exp_map, i.e. everything inside
 *                          SE3DeformationField.forward (nerfstudio/field_components/deformation_field.py:134-166),
 *                          HashEnsemble.forward (nerfstudio/field_components/hash_ensemble.py:93-158),
 *                          NeRSembleNeRFactoField.forward (nerfstudio/fields/nersemble_nerfacto_field.py:385-402)
 *                          and NeRSembleNGPModel.field_density_fn (nerfstudio/models/nersemble_instant_ngp.py:235-266)
 *   nsb_hash_blend_forward HashEnsemble.forward alone (component API)
 *   nsb_hash_blend_backward torch autograd through HashEnsemble.forward alone (component API)
 *   nsb_composite_forward  nerfacc.pack_info / render_weight_from_density + RGB/Depth/Accumulation/
 *                          Deformation renderers (nersemble_instant_ngp.py:325-343,359-362;
 *                          nerfstudio/model_components/nersemble_deformation_renderer.py:10-29)
 *   nsb_march_*            nerfacc OccGridEstimator.sampling -> traverse_grids
 *                          (nerfstudio/model_components/nersemble_volumetric_sampler.py:95-108)
 *   nsb_visibility_*       nerfacc render_visibility_from_density (the training pre-pass of sampling())
 *   nsb_composite_backward / nsb_field_backward / nsb_deform_backward
 *                          torch autograd through all of the above (training; with per-sample conditioning codes also
 *                          for the stand-alone field and deformation modules of the component API)
 *   nsb_table_adam_step    torch.optim.Adam on the 8 tcnn grid tensors (scripts/train/train_nersemble.py:243-247) and
 *                          tcnn's per-call fp32 -> fp16 cast of the table parameters
 */
#ifndef NSB_H
#define NSB_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NSB_VERSION 200
#define NSB_MAX_LEVELS 16
#define NSB_MEMBERS 32        /* ensemble members (hash_ensemble_config.n_hash_encodings) */
#define NSB_FEATS 2           /* features per member per level */
#define NSB_TILE 128          /* samples per CTA tile */
#define NSB_WARP_CODE_DIM 128 /* deformation warp-code width */
#define NSB_N_FREQ 7          /* SE3DeformationFieldConfig.n_freq_pos */

/* Hash-grid level table, computed on the host with tcnn's float32 formulas
 * (scale = exp2f(l*log2f(s))*base - 1, res = ceil(scale)+1, entries = min(round_up(res^3,8), 2^log2T)). */
typedef struct nsb_levels {
    int32_t n_levels;
    float scale[NSB_MAX_LEVELS];
    uint32_t res[NSB_MAX_LEVELS];
    uint32_t entries[NSB_MAX_LEVELS];
    uint32_t offset[NSB_MAX_LEVELS]; /* first entry of the level in the table */
    uint32_t hashed[NSB_MAX_LEVELS]; /* 1: XOR-prime hash, 0: dense stride index */
} nsb_levels;

/* Parameters of the field, in the native layouts (all DEVICE pointers). */
typedef struct nsb_field_params {
    const void *tables;        /* __half [total_entries][32 members][2 feats]: 128 B per entry */
    const float *deform_bias;  /* float [6*128 + 8]: stem biases, then v_bias(3), r_bias(3), 0, 0 */
    const void *deform_packed_tb;   /* fp16 deformation weights in MMA-B fragment order WITHOUT the warp-code columns of
                                       layers 0 and 4 (python: pack_deform_tb; nsb_deform_packed_bytes() bytes) */
    const float *deform_code_bias;  /* float [n_timesteps][2][128]: W_code(layer 0|4) . warp_code[t] + bias, fp32: the
                                       warp code only depends on the timestep, so its columns cost no tensor work
                                       (-26 % MACs).  Per-sample warp codes (component API): nsb_samples.sample_code_bias. */
    const void *deform_packed_umma; /* optional: the same deformation weights as wgmma B operands -- 14 blocks per tile in
                                       order of use (L0 | L1 x2 | L2 x2 | L3 x2 | L4 hidden x2, posenc | L5 x2 | heads x2), each
                                       [128 outputs x 64 inputs] fp16 (heads [16 x 64]) in K-major 8 x 16-byte core matrices
                                       (python: pack_deform_umma; nsb_deform_packed_umma_bytes()).  When set, the inference
                                       kernels run the deformation MLP on wgmma.mma_async (sm_90a warpgroup MMA). */
    const void *frame_table;   /* optional, float2 [n][total_entries]: the tables blended with the member weights of one or
                                  more timesteps (nsb_blend_tables).  The gather then reads 8 B per corner instead of a
                                  128 B line.  Used by the wgmma inference kernels.  With frame_stride == 0 it is ONE
                                  timestep's table and only valid when EVERY sample of the call has that timestep (one
                                  camera frame: a 50 MB table that stays in L2). */
    int64_t frame_stride;      /* entries between consecutive timesteps' tables in frame_table: a sample of timestep t
                                  gathers from frame_table + t * frame_stride.  total_entries for a stack of all
                                  n_timesteps tables (rays of mixed timesteps); 0 for one frame table.
                                  frame_stride * n_timesteps must be < 2^32. */
    const void *field_packed;  /* fp16 mlp_base + mlp_head weights in MMA-B fragment order */
    const void *warp_codes;    /* __half [n_timesteps][128]  (time_embedding_deformation) */
    const float *blend_codes;  /* float  [n_timesteps][32]   (time_embedding) */
    int32_t n_timesteps;
    float aabb[6];             /* min xyz, max xyz */
    nsb_levels levels;
} nsb_field_params;

/* Per-call options of the field evaluation. */
typedef struct nsb_field_opts {
    /* effective blend weight of member h: cw[h] = code[h]*cw_scale[h] + cw_bias[h]
     * (window, disable_initial_hash_ensemble and soft transition folded in on the host:
     *  hash_ensemble.py:119-139) */
    float cw_scale[NSB_MEMBERS];
    float cw_bias[NSB_MEMBERS];
    float pe_window[8];       /* Hann window of the 7 posenc bands (windowed_nerf_encoding.py:76-92); 1 if None */
    int32_t use_deformation;  /* config.use_deformation_field */
    int32_t compute_rgb;      /* 0: density only (field_density_fn) */
} nsb_field_opts;

/* Sample sources.  Either ray-based packed samples (positions = o + d*(ts+te)/2, per-ray times)
 * or explicit positions with per-sample times (density_fn / occupancy update). */
typedef struct nsb_samples {
    int64_t n_samples;
    /* ray-based */
    const float *origins;      /* [n_rays][3] */
    const float *directions;   /* [n_rays][3] */
    const float *ray_times;    /* [n_rays] in [0,1] or NULL (timestep 0) */
    const float *t_starts;     /* [n_samples] */
    const float *t_ends;       /* [n_samples] */
    const int32_t *ray_indices;/* [n_samples] */
    /* explicit (used when origins == NULL) */
    const float *positions;    /* [n_samples][3] world */
    const float *sample_times; /* [n_samples] in [0,1] or NULL */
    const float *sample_directions; /* [n_samples][3] or NULL (density_fn uses ones: nersemble_nerfacto_field.py:240) */
    const int64_t *n_samples_dev;    /* optional DEVICE scalar: the packed sample count when only the device knows it (the
                                        sync-free training sampler); n_samples is then the capacity of the arrays */
    const void *given_feat;          /* optional __half [n_samples][32]: blended hash features already gathered for these
                                        samples (the density pre-pass of the training sampler, packed by
                                        nsb_visibility_compact); the kernel then skips the table gather entirely */
    /* optional per-sample conditioning overriding the time-embedding tables (component APIs) */
    const float *sample_blend_codes; /* float  [n_samples][32] or NULL */
    const float *sample_code_bias;   /* float [n_samples][2][128] or NULL: W_code(layer 0|4) . warp_code[sample] + bias
                                        (python: packing.deform_code_bias on the per-sample codes); <= 2^24 samples */
} nsb_samples;

typedef struct nsb_field_out {
    float *sigma;    /* [n_samples]     or NULL */
    float *rgb;      /* [n_samples][3]  or NULL (needs compute_rgb) */
    float *offsets;  /* [n_samples][3]  or NULL: p' - p in normalised-aabb units (deformation_field.py:148-166) */
    void *feat;      /* __half [n_samples][32] blended hash features or NULL */
    float *xs;       /* [n_samples][4] or NULL: normalised warped position fed to the hash grids (0 outside the box),
                        w = in-box selector.  Saved by the training forward for nsb_field_backward. */
    void *deform_acts; /* NULL or uint4 [n_tiles][8 warps][6 layers][8 k-tiles][32 lanes]: fp16 outputs of the 6 stem
                        layers in MMA A-fragment order (16 rows per warp), saved by the training forward for
                        nsb_deform_backward (the reference keeps the same activations for autograd). */
    void *deform_enc;  /* NULL or uint4 [n_tiles][8 warps][3 k-tiles][32 lanes]: windowed posenc fragments */
    void *corner_vals; /* NULL or __half2 [n_samples][16 levels][8 corners]: member-blended (f0, f1) of every gathered
                          corner before the trilinear weight; saved by the training forward so that nsb_field_backward
                          computes the position gradient without gathering the table lines again */
} nsb_field_out;

int nsb_version(void);
const char *nsb_last_error(void);

/* Sizes (bytes) of the packed weight buffers the python packer must produce. */
size_t nsb_deform_packed_bytes(void);
size_t nsb_deform_packed_umma_bytes(void);
/* Frame tables of n_timesteps consecutive timesteps first_timestep, first_timestep + 1, ...:
 *   out[i][e] = sum_m (blend_codes[first_timestep + i][m] * cw_scale[m] + cw_bias[m]) * tables[e][m][:]
 * (float2 [n_timesteps][n_entries], fp32 accumulation) -- HashEnsemble.forward's member blend (hash_ensemble.py:119-139)
 * hoisted out of the per-sample path (nsb_field_params.frame_table / frame_stride).  One pass: every 128 B line is read
 * once for all n_timesteps outputs, and slice i is bit-identical to the n_timesteps = 1 call for that timestep. */
int nsb_blend_tables(const nsb_field_params *params, const nsb_field_opts *opts, int32_t first_timestep,
                     int32_t n_timesteps, int64_t n_entries, void *out, void *stream);
size_t nsb_field_packed_bytes(void);

/* Fused per-sample field evaluation (deformation MLP -> SE(3) warp -> 32-member hash ensemble
 * gather+blend -> density MLP -> colour MLP).  One persistent kernel. */
int nsb_field_forward(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                      const nsb_field_out *out, void *stream);

/* HashEnsemble.forward: x [n][3] float in [0,1), code float [n][32] -> out __half/float [n][32].
 * out_is_half: 1 -> __half output, 0 -> float. */
int nsb_hash_blend_forward(const nsb_field_params *params, const nsb_field_opts *opts, const float *x,
                           const float *codes, int64_t n, void *out, int32_t out_is_half, void *stream);
/* Backward of nsb_hash_blend_forward for d_out float [n][32] (output order l*2+f), the same opts as the forward:
 *   d_tables fp32 [total_entries][32][2], ACCUMULATED (+=), NULL: skip;  d_codes [n][32] and d_x [n][3], written, NULL: skip.
 * The blend weights are rounded to fp16 like the forward's; a member whose weight the window fixes (w == 1 with
 * disable_initial_hash_ensemble) gets a code gradient of exactly 0. */
int nsb_hash_blend_backward(const nsb_field_params *params, const nsb_field_opts *opts, const float *x,
                            const float *codes, int64_t n, const float *d_out, float *d_tables, float *d_codes,
                            float *d_x, void *stream);

/* Alpha compositing of packed samples. packed_info int64 [n_rays][2] = (start, count). */
typedef struct nsb_composite_args {
    int64_t n_rays, n_samples;
    const int64_t *packed_info;
    const float *t_starts, *t_ends, *sigma, *rgb, *offsets; /* offsets may be NULL */
    int32_t training;     /* 0: eval (nan_to_num before, clamp[0,1] after) */
    float *out_rgb;       /* [n_rays][3] white background */
    float *out_acc;       /* [n_rays] */
    float *out_depth;     /* [n_rays] expected depth, clipped to [min(steps), max(steps)] */
    float *out_deform;    /* [n_rays][3] or NULL */
    float *out_weights;   /* [n_samples] or NULL */
    uint32_t *workspace;  /* 2 uint32 (ordered-float min/max of sample midpoints) */
} nsb_composite_args;
int nsb_composite_forward(const nsb_composite_args *args, void *stream);

/* Backward of nsb_composite_forward (training mode): gradients w.r.t. per-sample sigma and rgb.
 * d_weights (the losses that act on per-sample weights: empty/near/distortion, models/base.py:136-249)
 * may be NULL.  `workspace` must be the one nsb_composite_forward filled (depth clip range). */
typedef struct nsb_composite_bwd_args {
    int64_t n_rays, n_samples;
    const int64_t *packed_info;
    const float *t_starts, *t_ends, *sigma, *rgb;
    const float *d_out_rgb;    /* [n_rays][3] */
    const float *d_out_acc;    /* [n_rays]    or NULL */
    const float *d_out_depth;  /* [n_rays]    or NULL */
    const float *d_weights;    /* [n_samples] or NULL */
    const uint32_t *workspace;
    float *d_sigma;            /* [n_samples] out */
    float *d_rgb;              /* [n_samples][3] out */
} nsb_composite_bwd_args;
int nsb_composite_backward(const nsb_composite_bwd_args *args, void *stream);

/* Backward of the field MLPs + hash ensemble (replaces the autograd of tcnn mlp_base/mlp_head, the einsum blend
 * and tcnn's kernel_grid_backward: nersemble_nerfacto_field.py:285-301,377; hash_ensemble.py:102-156).
 * Inputs saved by the training forward: feat, xs, sigma, rgb.  Gradients are ACCUMULATED (+=) into the fp32
 * outputs, which the caller zeroes.  The deformation field's backward is not part of this entry point. */
typedef struct nsb_field_bwd_args {
    const void *field_packed_t;   /* fp16 TRANSPOSED field weights in MMA-B fragment order (python: pack_field_bwd) */
    const void *feat;             /* __half [n][32] */
    const float *xs;              /* [n][4] */
    const float *sigma;           /* [n] */
    const float *rgb;             /* [n][3] (may be NULL when d_rgb is: density only) */
    const float *d_sigma;         /* [n] */
    const float *d_rgb;           /* [n][3] or NULL */
    float loss_scale;             /* MLP deltas are fp16 MMA operands: incoming grads are multiplied by this, outputs divided */
    float *d_feat;                /* [n][32] workspace/out: dL/d(blended features) */
    float *d_base_w;              /* [3072] tcnn mlp_base.params layout, += */
    float *d_head_w;              /* [7168] tcnn mlp_head.params layout, += */
    float *d_tables;              /* [total_entries][32][2] fp32, += (NULL: skip the table/code pass) */
    float *d_blend_codes;         /* [n_timesteps][32], += (NULL: skip) */
    float *d_xs;                  /* [n][3] out (NULL: skip): dL/d(normalised warped position), tcnn's
                                     kernel_grid_backward_input; feeds the deformation-field backward */
    /* Rank-1 table-gradient path (table-indexed blend codes only).  The gradient of a table line is
     * cw_t[member] x (w_corner * dfeat[level, feat]): all samples of one timestep share cw_t, so the scatter only
     * accumulates the 2-vector per (timestep slot, line) -- 32x fewer atomics -- and nsb expands
     * d_tables[line][m][f] = sum_t cw_t[m] G[t][line][f] (and the time-code gradient) in one dense pass. */
    float *g_rank1;               /* workspace [n_slots][total_entries][2], zeroed by the caller; NULL: direct scatter */
    const int32_t *ts_slot;       /* [n_timesteps] -> slot in [0, n_slots) or -1 (timestep absent from this batch) */
    int32_t n_slots;
    const void *corner_vals;      /* NULL or nsb_field_out.corner_vals of the forward (rank-1 path: skips the re-gather) */
    float *cw_slots_out;          /* NULL or [n_slots][32] out: the effective (fp16-rounded) blend weights of each slot's
                                     timestep, exactly as the expansion uses them -- input of nsb_table_adam_step /
                                     nsb_rank1_expand when the caller defers the table gradient (d_tables == NULL) */
    float *d_sample_blend_codes;  /* [n][32] out or NULL: with nsb_samples.sample_blend_codes, each sample's blend-code
                                     gradient (written, not accumulated; direct scatter, d_blend_codes is not touched) */
} nsb_field_bwd_args;
int nsb_field_backward(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                       const nsb_field_bwd_args *args, void *stream);

/* Backward of the SE(3) deformation field (replaces the autograd of deformation_field.py:77-166, se3_exp_map and the
 * time_embedding_deformation lookup).  Needs the activations the training forward saved (nsb_field_out.deform_acts /
 * deform_enc) and dL/d(hash input position) from nsb_field_backward (d_xs).  fp32 gradients are ACCUMULATED (+=) in the
 * reference's parameter layouts (nn.Linear weight [out][in], input order of nerfstudio's MLP: layer 4 = [input 173 | hidden 128]). */
typedef struct nsb_deform_bwd_args {
    const void *deform_packed_t;  /* fp16 TRANSPOSED stem/head weights in MMA-B fragment order (python: pack_deform_bwd) */
    const void *deform_acts;
    const void *deform_enc;
    const float *d_xs;            /* [n][3] */
    float loss_scale;
    float *d_stem_w[6];           /* [128][173], 3 x [128][128], [128][301], [128][128] */
    float *d_stem_b;              /* [6][128] */
    float *d_r_w, *d_r_b;         /* [3][128], [3] */
    float *d_v_w, *d_v_b;         /* [3][128], [3] */
    float *d_warp_codes;          /* [n_timesteps][128] or NULL */
    void *dw_workspace;           /* nsb_deform_bwd_workspace_bytes() of scratch (need not be zeroed): per-CTA private
                                     weight-gradient accumulators, summed into d_stem_w at the end of the call */
    /* Per-sample warp codes (component API; the forward took them as nsb_samples.sample_code_bias).  When set, the code
       columns of d_stem_w[0] / d_stem_w[4] use these codes, params->warp_codes and d_warp_codes are not used, and
       d_sample_warp_codes (NULL: skip) receives each sample's code gradient, ACCUMULATED (+=) without atomics. */
    const void *sample_warp_codes;  /* __half [n][128] or NULL */
    float *d_sample_warp_codes;     /* [n][128] */
} nsb_deform_bwd_args;
size_t nsb_deform_packed_t_bytes(void);
size_t nsb_deform_bwd_workspace_bytes(void);
int nsb_deform_backward(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                        const nsb_deform_bwd_args *args, void *stream);

/* Fused hash-table optimiser step.  Replaces, for the table parameter only, what the reference's training loop does
 * with torch: materialise the dense fp32 gradient of the 8 tcnn grids, run torch.optim.Adam over it (nerfstudio
 * AdamOptimizerConfig, eps 1e-15: train_nersemble.py optimizers["fields"]) and let tcnn re-read the parameters.  One
 * pass over the table: gradient line = sum_slots cw_slot[member] x G[slot][line][feat] (rank-1 expansion of the
 * scatter workspace nsb_field_backward filled) and/or a dense fp32 gradient, times grad_scale; torch.optim.Adam's
 * update (lerp form of exp_avg, bias corrections passed in, no amsgrad); the fp16 copy the forward kernels gather is
 * rewritten in the same pass.  Every line is updated (Adam's moments decay where the gradient is zero, like torch). */
typedef struct nsb_table_adam_args {
    int64_t total_entries;
    float *tables;            /* fp32 master [E][32][2], in place */
    float *exp_avg;           /* [E][32][2], in place */
    float *exp_avg_sq;        /* [E][32][2], in place */
    void *tables_half;        /* __half [E][32][2] out, or NULL */
    const float *grad;        /* dense fp32 gradient [E][32][2] or NULL */
    const float *g_rank1;     /* [n_slots][E][2] or NULL */
    const float *cw_slots;    /* [n_slots][32] (nsb_field_bwd_args.cw_slots_out) */
    int32_t n_slots;          /* <= 32 */
    float grad_scale;         /* e.g. 1 / world_size */
    float lr, beta1, beta2, eps, weight_decay;
    float bias_correction1;   /* 1 - beta1^step */
    float bias_correction2;   /* 1 - beta2^step */
    /* The scalars of torch.optim.Adam's update, each formed in double precision on the host and rounded once to float,
       as torch forms them: the table step is then bit-identical to torch's foreach Adam for the same gradient. */
    float step_size;          /* lr / bias_correction1 */
    float bias_correction2_sqrt; /* bias_correction2 ** 0.5 */
    float one_minus_beta1, one_minus_beta2;
} nsb_table_adam_args;
int nsb_table_adam_step(const nsb_table_adam_args *args, void *stream);

/* d_tables[line][m][f] += grad_scale * sum_slots cw_slot[m] * G[slot][line][f]: the deferred expansion alone (used when
 * a deferred gradient has to become a dense .grad after all: gradient accumulation, dense all-reduce). */
int nsb_rank1_expand(const float *g_rank1, const float *cw_slots, int32_t n_slots, int64_t total_entries,
                     float grad_scale, float *d_tables, void *stream);

/* The six training losses (reference: models/base.py:90-249 via models/nersemble_instant_ngp.py:366-407, and
 * torch_efficient_distloss.flatten_eff_distloss) and their gradients w.r.t. the render outputs, fused: two launches
 * forward, one backward, no host synchronisation (formulas in csrc/nsb_losses.cu).  A lambda of 0 (or alpha /
 * depth_target == NULL) switches the corresponding term off; its value is then 0. */
typedef struct nsb_loss_args {
    int64_t n_rays, n_samples;
    const int64_t *packed_info;   /* [n_rays][2] */
    const float *t_starts, *t_ends, *weights;   /* [n_samples] */
    const float *rgb, *acc, *depth;             /* [n_rays][3], [n_rays], [n_rays] */
    const float *image;           /* [n_rays][3] ground truth */
    const float *alpha;           /* [n_rays] in [0,1] (alpha_map / 255) or NULL */
    const float *depth_target;    /* [n_rays] (0 = no depth) or NULL: empty / near / depth losses */
    int32_t use_masked_rgb;
    float alpha_mask_threshold;
    float lambda_alpha, lambda_empty, lambda_near, lambda_depth, lambda_dist;
    float eps_depth;
    int64_t dist_max_rays;
    double *accum;                /* [16] workspace (forward zeroes it) */
    float *values;                /* [6] out: rgb, alpha, empty, near, depth, dist loss values */
    float *coef;                  /* [8] out (forward) / in (backward): per-element gradient factors */
    const float *upstream;        /* backward: [6] dL/d(values) */
    float *d_rgb, *d_acc, *d_depth, *d_weights;   /* backward out: [n_rays][3], [n_rays], [n_rays], [n_samples] */
} nsb_loss_args;
int nsb_losses_forward(const nsb_loss_args *args, void *stream);
int nsb_losses_backward(const nsb_loss_args *args, void *stream);

/* Fixed-stride marcher (BASELINE configs 1/2): n_per_ray intervals of `step` from max(t_enter, near). */
int nsb_march_fixed(const float *origins, const float *directions, int64_t n_rays, const float *aabb6,
                    int32_t n_per_ray, float step, float near_plane, float *t_starts, float *t_ends,
                    int32_t *ray_indices, int64_t *packed_info, void *stream);

/* Occupancy-grid marcher (nerfacc traverse_grids, levels grids of res^3 bools).
 * Pass 1 (t_starts == NULL): writes counts[n_rays].  Pass 2: fills packed outputs at offsets[ray]. */
typedef struct nsb_march_args {
    int64_t n_rays;
    const float *origins, *directions;
    const float *near_planes, *far_planes; /* [n_rays] (jitter already added) */
    const uint8_t *binaries;               /* [levels][res][res][res] */
    const float *aabbs;                    /* [levels][6] */
    int32_t levels, res;
    float step, cone_angle;
    int32_t *counts;                       /* pass 1 out */
    const int64_t *offsets;                /* pass 2 in: exclusive scan of counts */
    float *t_starts, *t_ends;              /* pass 2 out */
    int32_t *ray_indices;                  /* pass 2 out */
} nsb_march_args;
int nsb_march_occupancy(const nsb_march_args *args, void *stream);

/* Visibility filter of the training pre-pass: keep = (T >= early_stop_eps) & (alpha >= alpha_thre). */
int nsb_visibility_mask(const int64_t *packed_info, int64_t n_rays, const float *t_starts, const float *t_ends,
                        const float *sigma, float early_stop_eps, float alpha_thre, uint8_t *mask,
                        int32_t *kept_counts, void *stream);

/* Occupancy-grid EMA update (nerfacc 0.5.2 estimators/occ_grid.py OccGridEstimator._update, called by
 * models/nersemble_instant_ngp.py:184-196 every 16 steps):
 *   occs[cell] = max(occs[cell] * ema_decay, occ_new[i])   for the evaluated cells cell_ids[i]
 *   thre = min(mean(occs[occs >= 0]), occ_thre);  binaries = occs > thre
 * cell_ids may repeat (uniform + occupied sampling): upstream's indexed assignment keeps the value of an unspecified
 * one of the duplicates; here a repeated cell deterministically gets max(old * decay, max_i occ_new[i]) -- the result
 * of the duplicate with the largest occ_new writing last.  scratch: float [n_cells] + double [2], caller-provided. */
int nsb_occ_update(float *occs, uint8_t *binaries, int64_t n_cells, const int64_t *cell_ids, const float *occ_new,
                   int64_t n, float ema_decay, float occ_thre, void *scratch, void *stream);
size_t nsb_occ_update_scratch_bytes(int64_t n_cells);

/* Fused inference render (SURVEY 8b `nsb_render_forward`; models/nersemble_instant_ngp.py:280-364 in eval mode):
 * sampler -> fused field kernel (deformation MLP, hash ensemble, density / colour MLPs) -> alpha compositing + global
 * depth clip, as phases of one persistent cooperative kernel (grid = number of SMs) separated by grid-wide barriers.
 * The fixed-stride march is a phase of that kernel; the nerfacc occupancy march (count -> scan -> fill, or one traversal
 * into per-ray slots) is a cooperative launch of its own just before it.  The packed-sample count never
 * leaves the device, so the call is free of host synchronisation; the per-sample arrays live in a caller-provided
 * workspace of `capacity` samples (an upper bound such as n_rays * ceil(aabb diagonal / step); if the march produces
 * more, the samples beyond it are dropped and `status` in the workspace header is set to 1).
 * Same device code as nsb_march_* / nsb_field_forward / nsb_composite_forward: results are bit-identical to that path. */
typedef struct nsb_render_args {
    int64_t n_rays;
    const float *origins, *directions; /* [n_rays][3] */
    const float *ray_times;            /* [n_rays] in [0,1] or NULL */
    int32_t sampler;                   /* 0: fixed-stride march (n_per_ray steps from max(t_enter, near_plane)); 1: occupancy
                                          march; any other value is rejected */
    int32_t n_per_ray;                 /* sampler 0 */
    float near_plane;                  /* sampler 0 */
    const float *near_planes, *far_planes; /* sampler 1: [n_rays] (jitter already added) */
    const uint8_t *binaries;           /* sampler 1: [levels][res][res][res] */
    const float *aabbs;                /* sampler 1: [levels][6] */
    int32_t levels, res;
    float step, cone_angle;
    int32_t training;                  /* compositing mode (0: eval nan_to_num / clamp) */
    int64_t capacity;                  /* samples the per-sample arrays below can hold */
    float *t_starts, *t_ends;          /* [capacity] out */
    int32_t *ray_indices;              /* [capacity] out */
    float *sigma, *rgb, *offsets;      /* [capacity], [capacity][3], [capacity][3] out (offsets NULL iff no deformation) */
    float *weights;                    /* [capacity] out or NULL */
    int64_t *packed_info;              /* [n_rays][2] out: (start, count) */
    float *out_rgb, *out_acc, *out_depth, *out_deform; /* [n_rays][3], [n_rays], [n_rays], [n_rays][3] | NULL */
    void *workspace;                   /* nsb_render_workspace_bytes(n_rays) bytes; header = nsb_render_ws_header */
    float *march_scratch;              /* sampler 1, optional: float [2][capacity].  With it the occupancy grid is traversed
                                          ONCE (samples land in per-ray slots of capacity / n_rays entries, then a coalesced
                                          copy packs them) instead of twice (count, fill): the DDA is a dependent chain per
                                          ray and dominates the march (4096 rays: 439 -> ~230 us).  A ray with more samples
                                          than its slot is truncated and status set to 1. */
} nsb_render_args;
typedef struct nsb_render_ws_header {  /* first 64 bytes of the workspace; n_total / status are results */
    uint32_t barrier;                  /* grid-barrier arrival counter (the call zeroes it) */
    uint32_t depth_range[2];           /* ordered-int min / max of the sample midpoints */
    int32_t status;                    /* 0 ok, 1 capacity exceeded */
    int64_t n_total;                   /* packed samples the march produced */
    int64_t reserved[5];
} nsb_render_ws_header;
size_t nsb_render_workspace_bytes(int64_t n_rays);
int nsb_render_forward(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_render_args *args, void *stream);

/* Surface normals of the density field (nerfstudio Field.get_normals, used by NeRSembleNeRFactoField.forward with
 * compute_normals=True: nerfstudio/fields/nersemble_nerfacto_field.py:385-402) and their per-ray composite
 * (NormalsRenderer with normalize=True), for samples the field or render kernels already evaluated:
 *   n = -normalize(grad_scale * d h0 / d x),  normalize(v) = v / max(|v|, 1e-12)
 * h0 = mlp_base output 0 before trunc_exp; x = the normalised hash-input position after the in-box selector (0 outside
 * the box: such a sample gets the gradient at the box origin), formed exactly as the field kernels form it (with offsets,
 * the normalised offsets added to the world position).  With deformation these are canonical-space normals.  The gather
 * reads the tables the field kernels read for the same params / samples: frame_table (one frame or a timestep stack),
 * else the 128 B lines with sample_blend_codes or the timestep's blend codes.  Not differentiable.
 *   out_normals[r] = v / (|v| + 1e-10), v = sum over the ray's packed_info segment of weights[i] * normals[i], summed
 * in a fixed order (bit-identical from run to run).  Samples beyond *n_samples_dev (when given) are not touched. */
typedef struct {
    const float *offsets;        /* [n][3] or NULL (no deformation): the offsets the field / render kernels wrote */
    float grad_scale[3];          /* per-axis factor on d h0 / d x before normalising: 1 (normalised space, the field API)
                                     or 1 / aabb extent (world space, rendered normals) */
    const int64_t *packed_info;   /* [n_rays][2] (start, count), needed for out_normals */
    int64_t n_rays;
    const float *weights;         /* [n] render weights, needed for out_normals */
    float *normals;               /* [n][3] out; NULL: nothing is computed (required for out_normals) */
    float *out_normals;           /* [n_rays][3] out or NULL */
} nsb_normals_args;
int nsb_normals_forward(const nsb_field_params *params, const nsb_field_opts *opts, const nsb_samples *samples,
                        const nsb_normals_args *args, void *stream);

/* Training sampler WITHOUT host synchronisation (model_components/nersemble_volumetric_sampler.py:95-108 around nerfacc
 * OccGridEstimator.sampling): (1) nsb_march_occupancy_packed = count/scan/fill of nsb_march_occupancy as ONE cooperative
 * launch, the candidate count stays in the workspace header; (2) the caller evaluates the candidates' density with
 * nsb_field_forward(samples->n_samples_dev = &header.n_total); (3) nsb_visibility_compact applies nerfacc's
 * render_visibility_from_density, mask = (T >= early_stop_eps) & (alpha >= min(alpha_thre, *alpha_thre_cap)), and packs
 * the surviving samples (plus optional per-sample payload rows of the pre-pass) -- mask | scan | copy in one cooperative
 * launch; the kept count lands in ITS workspace header. */
int nsb_march_occupancy_packed(const nsb_march_args *args /* counts/offsets unused */, int64_t capacity, int64_t *packed_info,
                               void *workspace /* nsb_render_workspace_bytes(n_rays) */, float *scratch /* [2][capacity] or NULL */,
                               void *stream);
typedef struct nsb_vis_compact_args {
    int64_t n_rays, capacity;
    const int64_t *packed_info;            /* candidates [n_rays][2] */
    const float *t_starts, *t_ends, *sigma;
    const int32_t *ray_indices;
    float early_stop_eps, alpha_thre;
    const float *alpha_thre_cap;           /* device scalar (occs.mean()) or NULL */
    int64_t *out_packed_info;              /* [n_rays][2] */
    float *out_t_starts, *out_t_ends;      /* [capacity] */
    int32_t *out_ray_indices;
    /* optional payload rows that move with their sample (pre-pass reuse) */
    const void *feat; void *out_feat;                 /* __half [.][32] */
    const float *xs; float *out_xs;                   /* float [.][4] */
    const void *corner_vals; void *out_corner_vals;   /* __half2 [.][16][8] */
    void *workspace;                       /* nsb_render_workspace_bytes(n_rays): header.n_total = kept samples */
} nsb_vis_compact_args;
int nsb_visibility_compact(const nsb_vis_compact_args *args, void *stream);
size_t nsb_vis_compact_workspace_bytes(int64_t n_rays, int64_t capacity);

/* Training-batch assembly on the GPU (data/nersemble_pixel_sampler.py:23-69 + nerfstudio RayGenerator / Cameras
 * [PERSPECTIVE]): for each sampled pixel (image, y, x) the ray (origin, unit direction, pixel area, time, camera index)
 * and the supervision values gathered from an image cache resident in device memory.  One launch, no host round trip. */
typedef struct nsb_ray_batch_args {
    int64_t n_rays;
    const int64_t *indices;        /* [n_rays][3] (image, y, x) */
    int64_t height, width;         /* of every cached image */
    const int64_t *image_camera;   /* [n_images] camera of each image, or NULL (image == camera) */
    const float *image_times;      /* [n_images] time in [0,1] of each image, or NULL */
    const float *intrinsics;       /* [n_cameras][4] fx, fy, cx, cy */
    const float *camera_to_world;  /* [n_cameras][3][4] row-major */
    const uint8_t *images;         /* [n_images][H][W][3] or NULL */
    const uint8_t *alpha_maps;     /* [n_images][H][W]    or NULL */
    const float *depth_maps;       /* [n_images][H][W]    or NULL */
    float *origins, *directions;   /* [n_rays][3] out */
    float *pixel_area;             /* [n_rays] out or NULL */
    float *directions_norm;        /* [n_rays] out or NULL */
    float *times;                  /* [n_rays] out or NULL */
    int64_t *camera_indices;       /* [n_rays] out or NULL */
    float *out_image;              /* [n_rays][3] in [0,1] out or NULL */
    float *out_alpha;              /* [n_rays] in 0..255 out or NULL */
    float *out_depth;              /* [n_rays] out or NULL */
} nsb_ray_batch_args;
int nsb_ray_batch(const nsb_ray_batch_args *args, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NSB_H */
