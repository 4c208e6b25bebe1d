/*
 * difflinker_b200 -- C-ABI of the H100-native (sm_90a) DiffLinker denoising hot path.
 *
 * The reference (igashov/DiffLinker) is pure Python/PyTorch and has no FFI; the boundary this library
 * replaces is the set of Python call sites listed below (SURVEY.md section 8(b)).  Every entry point is
 * extern "C", takes plain pointers/sizes (no torch types), is stream-ordered and non-blocking unless
 * stated, and returns a dl_status.  One engine per GPU, used from one host thread at a time.
 *
 *   reference interface (file:line)                      entry point here
 *   ---------------------------------------------------  ------------------------------------------
 *   Dynamics.__init__            src/egnn.py:324-372     dl_create / dl_destroy
 *     tanh, sin_embedding, aggregation_method  egnn.py:101-106,281-292,304-320  dl_create_ex (dl_egnn_options)
 *   Dynamics.load_state_dict     (ckpt keys, SURVEY 8b)  dl_set_weight / dl_finalize_weights
 *   Dynamics.forward             src/egnn.py:374-447     dl_dynamics_forward (+ _host)
 *   DynamicsWithPockets.forward  src/egnn.py:471-552     dl_dynamics_forward with graph_type != DL_GRAPH_FC
 *   EDM.sample_chain             src/edm.py:126-176      dl_sample_chain (+ _host)
 *     sample_p_zs_given_zt_only_linker  edm.py:178-208
 *     sample_p_xh_given_z0_only_linker  edm.py:210-235
 *   InpaintingEDM.sample_chain   src/edm.py:549-612      dl_sample_chain (+ _rng) with DL_SAMPLER_INPAINT
 *   either, one seed per molecule (no reference API)     dl_sample_chain_seeded
 *   EDM, from q(z_t0 | x) of a known linker (edm.py:67-74) dl_set_start_step, then any dl_sample_chain* entry point
 *     at step t0 (partial diffusion, no reference API)
 *     ... at one step t0[b] per molecule                 dl_set_start_steps, then the per-row entry points
 *   EDM, deterministic DDIM or DPM-Solver++(2M) steps   dl_set_solver, then any dl_sample_chain* entry point
 *     instead of p(z_s | z_t) (no reference API)
 *   EDM, keeping given linker atoms and sampling the    dl_set_fixed_atoms before each dl_sample_chain* call
 *     rest (replacement, RePaint without re-noising passes; no reference API)
 *   EDM, with linker atoms of allowed elements only      dl_set_linker_types before each dl_sample_chain* call
 *     (the data prediction projected; no reference API)
 *   InpaintingEDM, r RePaint passes per step            dl_set_resamplings, then any dl_sample_chain* entry point
 *     (DiffSBDD's inpaint(..., resamplings=r), no reference API)
 *   either, resampling only the molecules that diverged  dl_sample_chain_retry, dl_retry_seed, dl_last_retry_ms
 *     (the reference's callers resample the whole batch, generate.py:153-161)
 *   either, also resampling the molecules that are      dl_sample_chain_retry with dl_molecule_checks, dl_molecule_check
 *     disconnected (is_connected, src/metrics.py:20-27, on the molecules of src/lightning.py:364-377) or have an atom
 *     beyond its valence (the explicit-valence part of validity, src/metrics.py:12-17; see dl_molecule_checks)
 *   either on pocket graphs, also resampling the        dl_sample_chain_retry with DL_CHECK_CLASH, dl_clash_check
 *     molecules whose linker clashes with the pocket (no reference API; see dl_molecule_checks)
 *   EDM on pocket graphs, pushing linker atoms out of     dl_set_clash_guidance, then any dl_sample_chain* entry point;
 *     the pocket during the last K steps (no reference   dl_clash_guide
 *     API; see dl_set_clash_guidance)
 *   either, also resampling the molecules that repeat   dl_sample_chain_retry with DL_CHECK_UNIQUE, dl_molecule_hash
 *     a batch-mate (uniqueness, compute_metrics.py; see DL_CHECK_UNIQUE)
 *   either, also resampling the molecules whose linker   dl_sample_chain_retry_sets with DL_CHECK_NOVEL (known set) or
 *     is known, or that repeat an earlier call's          DL_CHECK_UNIQUE (seen set); dl_molecule_hash over the linker rows
 *     (novelty, compute_metrics.py; see DL_CHECK_NOVEL)   and dl_novel_check
 *   either, also resampling the molecules whose linker   dl_sample_chain_retry with DL_CHECK_RINGS, dl_set_ring_sizes,
 *     closes a ring of a size not allowed (see            dl_last_ring_sizes, dl_ring_check
 *     DL_CHECK_RINGS)
 *   either, also resampling the molecules whose linker   dl_sample_chain_retry with DL_CHECK_ANCHORS, dl_set_anchors,
 *     does not attach at the given anchors (--anchors,     dl_anchor_check
 *     generate.py:130-140; find_exit, compute_metrics.py;
 *     see DL_CHECK_ANCHORS)
 *   SizeClassifier.forward       src/linker_size_lightning.py:83-110  dl_sizegnn_create/.../dl_sizegnn_forward
 *   softmax + Categorical.sample of a size model (generate.py:88-99), from dl_size_draw, dl_size_uniform
 *     the molecule's seed, and redrawn in the recovery rounds             dl_sample_chain_retry with dl_size_redraw
 *   build_xae_molecule           src/molecule_builder.py:44-102       dl_bond_orders
 *   frame restore + .xyz text    generate.py:163-171, src/visualizer.py:14-31   dl_restore_frame, dl_format_xyz
 *   utils.FoundNaNException      src/utils.py:274-289    DL_NAN_DETECTED + per-molecule nan_flags
 *
 * Memory: all `const` device pointers are caller-owned and only read; outputs are caller-owned.
 * Floats are fp32, masks int8 exactly as datasets.collate produces them (src/const.py:6-7,
 * src/datasets.py:353-369: edge_mask values are {0,-1,-2}, self-loops live).
 */
#ifndef DIFFLINKER_B200_H_
#define DIFFLINKER_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dl_engine dl_engine; /* opaque */

typedef enum dl_status {
  DL_OK = 0,
  DL_NAN_DETECTED = 1,        /* dynamics produced NaN: see nan_flags (bit0 = coordinates, bit1 = features) */
  DL_ERR_INVALID = -1,        /* bad argument / unsupported configuration */
  DL_ERR_CUDA = -2,           /* CUDA runtime error; dl_last_error() has the text */
  DL_ERR_WEIGHTS = -3,        /* unknown / missing / wrongly sized weight */
  DL_ERR_UNSUPPORTED = -4
} dl_status;

enum { DL_GRAPH_FC = 0, DL_GRAPH_4A = 1, DL_GRAPH_FC_4A = 2, DL_GRAPH_FC_10A_4A = 3 };
enum { DL_EDGE_AUTO = 0, DL_EDGE_SIMT = 1, DL_EDGE_WGMMA = 2 };
enum { DL_SAMPLER_LINKER = 0, DL_SAMPLER_INPAINT = 1 };
enum { DL_AGGR_SUM = 0, DL_AGGR_MEAN = 1 };
enum { DL_SOLVER_ANCESTRAL = 0, DL_SOLVER_DDIM = 1, DL_SOLVER_DPMPP_2M = 2 };   /* dl_set_solver */

/* Mirrors the kwargs of Dynamics.__init__ (src/egnn.py:324-329) that reach the hot path. */
typedef struct dl_config {
  int32_t n_dims;               /* 3 */
  int32_t in_node_nf;           /* F: width of the atom-feature block of xh (one-hot [+ charge]) */
  int32_t context_node_nf;      /* C */
  int32_t hidden_nf;            /* H: must be 128 (every published config, configs/[all].yml `nf: 128`) */
  int32_t n_layers;             /* L equivariant blocks */
  int32_t inv_sublayers;        /* S GCLs per block */
  int32_t condition_time;       /* 0/1 */
  int32_t centering;            /* 0/1 (True only for inpainting models, lightning.py:99) */
  int32_t graph_type;           /* DL_GRAPH_* */
  int32_t device;               /* CUDA ordinal */
  int32_t edge_impl;            /* DL_EDGE_*: AUTO = wgmma tensor-core path */
  float norm_constant;          /* EquivariantBlock norm_constant (configs: 1e-6) */
  float normalization_factor;   /* 100 */
} dl_config;

/* Per-reverse-step scalars, computed by the caller with the reference's own formulae
 * (edm.py:369-403) so the device loop reproduces them bit-for-bit. Row r = 0..T-1 is reverse step
 * s = T-1-r; row T is the final p(x,h|z0) step. */
typedef struct dl_step_coef {
  float t;          /* value of the time feature fed to the dynamics ((s+1)/T, or 0 for the last row) */
  float a;          /* rows < T: alpha_{t|s}        ; row T: 1/alpha_0                         */
  float b;          /* rows < T: sigma2_{t|s}/alpha_{t|s}/sigma_t ; row T: sigma_0             */
  float c;          /* rows < T: sigma_{t|s}*sigma_s/sigma_t      ; row T: sigma_x = exp(gamma_0/2) */
  int32_t frame;    /* chain frame this step is the LAST writer of ((s*keep)//T, edm.py:162), or -1 */
  /* inpainting only (edm.py:650-670): q(z_s|z_t,x) on fragment atoms */
  float qa;         /* alpha_{t|s}*sigma_s^2/sigma_t^2 */
  float qb;         /* alpha_s*sigma2_{t|s}/sigma_t^2   */
  float pad;
} dl_step_coef;

/* EGNN options of the reference trainer (train_difflinker.py --tanh, --sin_embedding, --aggregation_method). */
typedef struct dl_egnn_options {
  int32_t tanh;                 /* 0/1: EquivariantUpdate bounds its update, trans = coord_diff * tanh(phi) * coords_range
                                   (egnn.py:101-106) */
  float coords_range;           /* 15: EGNN hands its own coords_range to every block (egnn.py:183,209) */
  int32_t sin_embedding;        /* 0/1: every edge MLP's first layer reads the 24 features [sin, cos](sqrt(r + 1e-8) f_k),
                                   f_k = 2 pi 4^k / 15, k < 6, of the block's and the input's radial r instead of the two
                                   radials (SinusoidsEmbeddingNew, egnn.py:281-292); edge_mlp.0 / coord_mlp.0 weights are then
                                   (H, 2H + 24) */
  int32_t aggregation;          /* DL_AGGR_SUM: sum / normalization_factor; DL_AGGR_MEAN: sum / the row's edge count in the
                                   reference's edge list (egnn.py:304-320) -- N on FC graphs, the cut-off degree (0 -> 1)
                                   on pocket graphs; normalization_factor is then unused */
} dl_egnn_options;

const char* dl_version(void);
const char* dl_last_error(void);

/* dl_create(cfg, out) is dl_create_ex(cfg, NULL, out); opts == NULL means {tanh 0, coords_range 15, sin_embedding 0,
 * DL_AGGR_SUM}, the reference's Dynamics defaults. */
dl_status dl_create(const dl_config* cfg, dl_engine** out);
dl_status dl_create_ex(const dl_config* cfg, const dl_egnn_options* opts, dl_engine** out);
dl_status dl_destroy(dl_engine* e);

/* `name` is the reference state_dict key relative to the Dynamics module, e.g.
 * "dynamics.e_block_0.gcl_1.edge_mlp.2.weight"; `data` is a HOST pointer to fp32 in the reference's
 * own (out,in) row-major layout.  Blocking (copies immediately). */
dl_status dl_set_weight(dl_engine* e, const char* name, const float* data, int64_t numel);
/* Verifies that every parameter of the configured architecture was provided, repacks them for the
 * kernels (k-major fp32 + fp16 hi/lo wgmma tiles) and uploads. Blocking. */
dl_status dl_finalize_weights(dl_engine* e);
/* Number of parameters (floats) the configured architecture expects; for load_state_dict checks. */
int64_t dl_expected_param_count(const dl_engine* e);

/*
 * One Dynamics.forward (egnn.py:374-447 / 471-552). DEVICE pointers.
 *   t          (t_numel) floats, t_numel == B or 1
 *   xh         (B,N,3+F)
 *   node_mask  (B,N) int8
 *   linker_mask (B,N) fp32 or NULL (inpainting, edm.py:505,632)
 *   edge_mask  FC graphs: (B*N*N) int8 or NULL (= all ones); pocket graphs: ignored (edges never cross
 *              molecules here; the reference's batch-id vector egnn.py:557,573 is implied by the layout)
 *   context    (B,N,C) fp32 or NULL when C == 0
 *   out        (B,N,3+F)
 *   nan_flags  (B) int32, written (not accumulated): bit0 NaN in vel, bit1 NaN in h; may be NULL
 * Enqueued on `stream` (a cudaStream_t); returns immediately.
 */
dl_status dl_dynamics_forward(dl_engine* e, int32_t B, int32_t N, const float* t, int32_t t_numel, const float* xh,
                              const int8_t* node_mask, const float* linker_mask, const int8_t* edge_mask,
                              const float* context, float* out, int32_t* nan_flags, void* stream);

/* Same with HOST buffers; copies in, runs, copies out, synchronises; returns DL_NAN_DETECTED if any
 * nan_flags entry is non-zero (nan_flags, if given, is a host array of B int32). */
dl_status dl_dynamics_forward_host(dl_engine* e, int32_t B, int32_t N, const float* t, int32_t t_numel,
                                   const float* xh, const int8_t* node_mask, const float* linker_mask,
                                   const int8_t* edge_mask, const float* context, float* out, int32_t* nan_flags);

/*
 * The whole reverse-diffusion loop (edm.py:126-235), on device, one CUDA-graph replay per step.
 *   xh         (B,N,3+F) normalised input (x/norm0, (h-bias)/norm1), DEVICE
 *   fragment_mask, linker_mask (B,N) fp32 DEVICE; node_mask (B,N) int8; edge_mask, context as above
 *   noise      (T+2,B,N,3+F) UNMASKED standard normal draws, DEVICE: slab 0 initialises the linker,
 *              slab 1+r feeds reverse step r, slab T+1 the final p(x|z0) draw -- i.e. the reference's
 *              torch.randn call order (edm.py:328-345).
 *              DL_SAMPLER_INPAINT (edm.py:549-727): (2T+3,B,N,3+F) PREPARED draws in the order the reference consumes
 *              them -- slab 0 initial z; slabs 1+2r / 2+2r the p(z_s|z_t) (all atoms) and q(z_s|z_t,x) (fragment atoms)
 *              draws of reverse step r; slabs 2T+1 / 2T+2 the final p(x|z0) and q(x|z0,x) draws -- each already
 *              multiplied by its mask with the coordinate part projected to zero centre of mass
 *              (utils.sample_center_gravity_zero_gaussian_with_mask, utils.py:158-168).  The engine must have been
 *              created with centering = 1 (lightning.py:99); all atoms move (the dynamics get linker_mask = NULL),
 *              the latent is re-centred every step (edm.py:592-594) and chain[0] mixes the two final variants by
 *              linker_mask / fragment_mask (edm.py:603-608).
 *   coef       (T+1) dl_step_coef, HOST
 *   norm       {norm_values[0], norm_values[1], norm_biases[1]} HOST (edm.py:347-355)
 *   chain      (keep_frames,B,N,3+F) DEVICE out; chain[0] holds final x and one-hot h (edm.py:174)
 *   nan_flags  (B) int32 DEVICE out: sticky bits as above, OR'ed with (first_nan_row+1)<<8
 * Enqueued on `stream`; the caller synchronises and inspects nan_flags (FoundNaNException mapping).
 */
dl_status dl_sample_chain(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                          const float* xh, const int8_t* node_mask, const float* fragment_mask,
                          const float* linker_mask, const int8_t* edge_mask, const float* context,
                          const float* noise, const dl_step_coef* coef, const float* norm, float* chain,
                          int32_t* nan_flags, void* stream);

/*
 * Same loop with the noise drawn ON THE DEVICE in the reference's stream order (edm.py:328-345, utils.py:189-192): per draw
 * torch.randn(B,N,3) then torch.randn(B,N,F). For a CUDA generator in state (seed, offset) those calls are Philox4x32-10
 * streams with a fixed thread -> element mapping (ATen DistributionTemplates.h); the kernels that consume the noise
 * regenerate exactly those numbers, so the result equals what `dl_sample_chain` returns for the tensor torch would have
 * drawn -- without the tensor ((T+2) B N (3+F) floats: 226 MB for B=256, N=40, T=500), its 2(T+2) launches and its
 * interleaving copy. A plain C caller can sample with nothing but a seed.
 *   seed, offset      the generator state on entry (torch.Generator.initial_seed() / get_offset(); offset % 4 == 0)
 *   offset_consumed   HOST out (may be NULL): what the draws consumed -- advance the generator by it
 * DL_SAMPLER_LINKER: T+2 raw draws, offset_consumed = (T+2) * per_draw.
 * DL_SAMPLER_INPAINT: the 2T+3 draws of InpaintingEDM in the same call order, offset_consumed = (2T+3) * per_draw. Each is
 *              masked and its coordinates are projected to zero centre of mass inside the per-molecule kernel, as the
 *              prepared slabs of dl_sample_chain describe (dl_noise_fill_inpaint writes them out). The raw draws are
 *              bit-identical to torch's; the projection sums each molecule in its own fixed order, so the coordinates
 *              agree with torch's projection to rounding (below 1e-6 absolute).
 */
dl_status dl_sample_chain_rng(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                              const float* xh, const int8_t* node_mask, const float* fragment_mask,
                              const float* linker_mask, const int8_t* edge_mask, const float* context, uint64_t seed,
                              uint64_t offset, uint64_t* offset_consumed, const dl_step_coef* coef, const float* norm,
                              float* chain, int32_t* nan_flags, void* stream);
/*
 * Same loop with a noise stream of each molecule's own: molecule b draws exactly what dl_sample_chain_rng gives a batch
 * holding only that molecule from generator state (seeds[b], 0) -- what the reference draws for it sampled alone after
 * torch.cuda.manual_seed(seeds[b]). So a molecule's chain depends neither on its batch-mates, nor on the batch size, its
 * row or the padding, and one molecule of a large run can be replayed on its own from its seed. Explicitly, element d of
 * atom n of molecule b in raw draw r (r < T+2 for DL_SAMPLER_LINKER, r < 2T+3 for DL_SAMPLER_INPAINT, in the call order of
 * dl_sample_chain_rng) is
 *     curandStatePhilox4_32_10_t st;
 *     curand_init(seeds[b], e, 8 * r + (d < 3 ? 0 : 4), &st);   value = curand_normal4(&st).x
 * with e = 3 n + d for the coordinates (d < 3) and e = F n + (d - 3) for the features. The inpainting sampler masks and
 * projects each draw per molecule as dl_sample_chain_rng does. This equals torch's own randn while N max(3, F) <= 2048 x the
 * device's SM count (about 17 k atoms on an H100); beyond that the formula above is the definition.
 *   seeds   (B) uint64 DEVICE, read while the call is enqueued (the loop reads the engine's copy); NULL is DL_ERR_INVALID.
 *           A torch seed s is reduced modulo 2^64, as torch.cuda.manual_seed does.
 * dl_set_noise_slice does not apply: the seeds already name the molecules, so a slice passes its rows of the seeds. Nothing
 * is consumed from any generator. Results also match across batches on the tensor-core path only while no sample diverges
 * far enough for the node GEMM to rescale a tile's fp16 operands (tiles span molecules; DESIGN.md section 6).
 */
dl_status dl_sample_chain_seeded(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                                 const float* xh, const int8_t* node_mask, const float* fragment_mask,
                                 const float* linker_mask, const int8_t* edge_mask, const float* context,
                                 const uint64_t* seeds, const dl_step_coef* coef, const float* norm, float* chain,
                                 int32_t* nan_flags, void* stream);
/*
 * The seed of attempt `attempt` of a molecule whose own seed is `seed` (dl_sample_chain_retry): attempt 0 (or below)
 * is `seed` itself; attempt a >= 1 is output a of a splitmix64 generator started from `seed`:
 *     z = seed + a * 0x9E3779B97F4A7C15;  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;
 *     z = (z ^ (z >> 27)) * 0x94D049BB133111EB;  return z ^ (z >> 31);            (all modulo 2^64)
 * For one attempt distinct seeds give distinct retry seeds. A pure host function.
 */
uint64_t dl_retry_seed(uint64_t seed, int32_t attempt);
/*
 * The checks a molecule can be put to, as data: connectivity and valence. Both are evaluated on the device, on the same atoms
 * and with the arithmetic of dl_bond_orders, on what src/lightning.py:364-377 builds from chain[0].
 *   atoms      molecule b's rows with node_mask != 0; on cut-off (pocket) graphs, graph_type != DL_GRAPH_FC, minus the pocket
 *              atoms, the rows whose last context column (pocket_only, src/egnn.py:486-487) is non-zero (lightning.py:372-374);
 *              inpainting models over all their atoms. Types are the first argmax of the first n_types feature columns, NaN
 *              winning.
 *   bond order of a pair: get_bond_order (src/molecule_builder.py:77-102) as dl_bond_orders evaluates it: 0, or 1 / 2 / 3 by
 *              100 |x_i - x_j| against thr1, thr2, thr3 [min type][max type] (a negative entry: the pair has no such bond).
 *              Atoms i and j bond iff the order is > 0, i.e. 100 |x_i - x_j| < thr1[min t][max t] and that entry >= 0:
 *              dl_bond_orders' E != 0 is exactly this relation.
 *   distance   |x_i - x_j| as torch.cdist measures it on the CPU over the n atoms the caller checks (the reference decides
 *              bonds after .cpu()), with i the later atom of the pair in the molecule's compacted atom order (dists[i, j],
 *              i > j). n <= 25: sqrt(fma(dz, dz, fma(dy, dy, dx * dx))). n > 25 (torch's _euclidean_dist):
 *              c = ((((-2 x_i0) x_j0 + (-2 x_i1) x_j1) + (-2 x_i2) x_j2) + |x_i|^2) + |x_j|^2, the second and third
 *              products fused, |x|^2 = (x0^2 + x1^2) + x2^2 rounded at each step; then a NaN-keeping clamp at 0 and a
 *              correctly rounded sqrt. n counts the checked atoms: connectivity, valence and the graph hash H use the atoms
 *              above, the linker hash L the linker atoms alone, dl_bond_orders the rows with node_mask != 0. So one pair can
 *              be decided differently in H and in L, or with and without the pocket rows, as it is in the reference.
 *              Residual: torch's CPU sqrt (MKL vsSqrt) rounds a fraction of a percent of its results one ulp away from the
 *              correctly rounded root (torch 2.11, MKL 2024.2, AVX-512), so a pair within one ulp of a threshold can be
 *              decided the other way there; the sgemm entries themselves matched this order bitwise.
 *   valence    of atom i: the integer sum of its pairs' bond orders over the other checked atoms. Pocket atoms are not
 *              partners either: src/lightning.py:372-374 drops them before the molecule is built.
 *   DL_CHECK_CONNECTED holds iff the graph of the atoms and their bonds has exactly one component (one atom is connected; no
 *              atom is not), i.e. len(Chem.GetMolFrags(mol)) == 1 for build_molecule's molecule: the reference's
 *              `is_connected` (src/metrics.py:20-27). Its AtomValenceException branch, which needs RDKit's valence model, is
 *              not reproduced; the reference applies is_connected to sanitized molecules only (metrics.py:103-104), and for
 *              those the two agree.
 *   DL_CHECK_VALENCE holds iff every checked atom has valence <= max_valence[type]. A molecule with no checked atom passes.
 * What is certain about DL_CHECK_VALENCE is just that: explicit valence within the caller's table, on dl_bond_orders' own
 * orders. build_molecule's molecules carry single, double and triple bonds only, no aromatic flags and no formal charges, so
 * an atom beyond its element's largest allowed valence is how Chem.SanitizeMol (is_valid, src/metrics.py:12-17) is expected
 * to reject them; that "SanitizeMol fails iff this check fails" has NOT been verified against RDKit. A caller with stricter
 * or looser chemistry passes their own table.
 *   DL_CHECK_CLASH (this library's own predicate; the reference has no clash test) holds iff no linker atom clashes with a
 *              pocket atom. Cut-off (pocket) graphs only, evaluated on chain[0] with the types above:
 *     linker atoms  rows with node_mask != 0, linker_mask != 0 and the last context column == 0. Fragment atoms are not
 *                   checked: they are inputs, which no resample moves.
 *     pocket atoms  rows with node_mask != 0 and the last context column != 0.
 *     clash         100 |x_i - x_j| in pm, in the direct form sqrt(fma(dz, dz, fma(dy, dy, dx * dx))) at every
 *                   atom count (the bond predicate's n <= 25 form, never torch.cdist's matmul form), is below
 *                   clash[min t][max t] of the caller's (n_types,n_types) table and that entry is >= 0; a negative entry means the pair never clashes (e.g. a
 *                   covalent warhead's element against the residue it binds).
 *   A molecule with no linker atom or no pocket atom passes. A NaN coordinate compares false and clashes with nothing
 *   (divergence is the NaN flag's business). The table is the struct's `clash` field (dl_clash_check takes it as an
 *   argument); molecule_builder.clash_table builds a default, 75% of the sum of the two elements' Bondi van der Waals
 *   radii, a common protein-ligand contact tolerance that has not been validated against any docking tool.
 */
/*
 *   DL_CHECK_UNIQUE (uniqueness among the samples of one input, compute_metrics.py) compares molecules with each other,
 *              by a graph hash of the atoms, types and bond orders above. With n atoms, t_i atom i's type, o_ij in {0,1,2,3}
 *              the bond order of the pair, mix(z) the splitmix64 finaliser of dl_size_uniform (z ^= z >> 30;
 *              z *= 0xBF58476D1CE4E5B9; z ^= z >> 27; z *= 0x94D049BB133111EB; z ^= z >> 31), TAG = 0x67726170682D776C
 *              ("graph-wl") and all arithmetic modulo 2^64:
 *                  c_0(i)     = mix(TAG ^ (t_i + 1))
 *                  c_{k+1}(i) = mix(c_k(i) + sum over j != i with o_ij > 0 of mix(c_k(j) + o_ij * 0x9E3779B97F4A7C15))
 *                  H          = mix(n + sum_i c_R(i)),   R = min(n, 64)          (no atom: H = mix(0) = 0)
 *              i.e. Weisfeiler-Lehman colour refinement with order-free sums. What it promises and what it does not:
 *                - isomorphic graphs (same elements, same bond orders) always hash equal, whatever the row order, pose
 *                  or padding;
 *                - non-isomorphic graphs can collide: 1-WL-equivalent pairs (e.g. decalin and bicyclopentyl) always do,
 *                  and a 64-bit collision is possible. A false duplicate costs one needless resample, never a returned
 *                  duplicate;
 *                - stereochemistry is ignored;
 *                - these are dl_bond_orders' graphs, not RDKit SMILES: two Kekule assignments of one aromatic ring are
 *                  different graphs. "Equal hash iff equal canonical SMILES" has NOT been verified against RDKit.
 *              The verdict, over the rows of one dl_sample_chain_retry call (the group is the whole call): after the first
 *              loop every row is a candidate; in recovery round a, the rows of that round's sub-batch are, each as the
 *              take rule left it. Keepers are the other rows that pass every required bit; eligible candidates are the
 *              finite ones with every other required bit. Candidate b gets DL_CHECK_UNIQUE iff its hash equals no
 *              keeper's and no eligible candidate b' < b has the same hash. Keepers never lose it, so rows that pass are
 *              not touched, and no two rows the call returns passing every required bit share a hash. A row that
 *              misses another bit blocks no one, so two such rows may both keep DL_CHECK_UNIQUE with one hash; they are
 *              resampled for the other bit anyway. dl_molecule_check refuses the bit (it checks each molecule alone); dl_molecule_hash gives the hashes, to compare across calls or
 *              devices.
 *              With a seen set (dl_hash_sets.seen: n_seen hashes in ascending unsigned order, duplicates allowed, e.g. the
 *              hashes an earlier call returned) the seen hashes count as keepers too: a candidate also loses the bit when
 *              its H is in the set. No returned row that passes every required bit then has a hash in the set, and no
 *              two such rows share a hash. Everything else about the verdict is unchanged.
 *   DL_CHECK_NOVEL (novelty, compute_metrics.py: the share of generated linkers that are not linkers of the training set)
 *              compares a molecule's linker with a caller's set of known linkers. The linker atoms of molecule b are its
 *              checked atoms (above) with linker_mask != 0; in the recovery rounds linker_mask is the sub-batch's, so a
 *              redrawn size counts the redrawn linker rows, as DL_CHECK_CLASH does. Its linker hash L_b is exactly the H
 *              of DL_CHECK_UNIQUE on the graph those atoms induce: the same types, the same dl_bond_orders orders, only
 *              the bonds between linker atoms -- the reference's linker, the molecule with every fragment atom removed
 *              (reformat_data_obabel.py). So L_b is dl_molecule_hash of the batch with node_mask replaced by
 *              node_mask AND linker_mask; a molecule with no linker atom has L = mix(0) = 0. The bit holds iff L_b is not
 *              in the caller's set (dl_hash_sets.known: n_known hashes in ascending unsigned order, duplicates allowed);
 *              an empty set passes every row. The limits are the hash's: novel means "by this hash, against linkers hashed
 *              the same way"; stereochemistry is ignored, there is no tautomer canonicalisation, 1-WL-equivalent graphs and
 *              64-bit collisions hash equal, and the hash has NOT been verified against RDKit canonical SMILES. A false
 *              "known" costs one needless resample and never returns a known linker. dl_molecule_check refuses the bit (it
 *              takes no linker_mask); dl_novel_check runs it on any batch, and dl_molecule_hash over node_mask AND
 *              linker_mask gives the same linker hashes.
 *   DL_CHECK_RINGS (a ring-size rule on the linker; compute_metrics.py reports rings after sampling) judges the smallest
 *              ring of every bond the linker takes part in:
 *     graph      the atoms and bonds of the checks above: checked atoms are rows with node_mask != 0, minus the pocket rows
 *                when drop_pocket applies; two atoms are bonded when dl_bond_orders gives an order > 0. Bonds are decided
 *                over all of the molecule's checked atoms, the same n that connectivity, valence and the graph hash H use
 *                (not the linker-only n of the linker hash L): the bond predicate switches form at n = 25, and rings
 *                through fragment atoms need the whole graph.
 *     linker atoms  checked atoms with linker_mask != 0; in the recovery rounds this is the sub-batch's linker_mask, as
 *                DL_CHECK_NOVEL reads it.
 *     smallest ring of a bond (u, v)  the number of atoms on a shortest cycle through that bond: 1 + the shortest-path
 *                length from u to v in the graph with that one bond removed. A bond on no cycle has no ring.
 *     ring-size mask of a molecule  a uint64: bit k is set iff some bond with at least one linker endpoint has a smallest
 *                ring of k atoms, for 3 <= k <= 62; bit 63 stands for any such ring of 63 or more atoms. Rings made only of
 *                fragment atoms are not judged: they are inputs, and no resample changes them (the reasoning of
 *                DL_CHECK_CLASH). A ring closed through both fragment and linker atoms is judged. A molecule with no linker
 *                bond on a cycle has mask 0.
 *              DL_CHECK_RINGS holds iff mask & ~allowed == 0, with `allowed` the caller's uint64 (dl_set_ring_sizes, or
 *              dl_ring_check's argument), whose bits 0-2 must be clear.
 *              Limits: these are rings of dl_bond_orders' graph. They are not RDKit's SSSR on OpenBabel-perceived bonds
 *              (reformat_data_obabel.py), and no claim is made that the result matches CalcNumRings or the reference's
 *              ring filter. A pair with a NaN coordinate compares false, so it is not bonded, as in the other checks.
 *              dl_molecule_check and dl_novel_check refuse the bit; dl_ring_check runs it on any batch.
 *   DL_CHECK_ANCHORS (the attachment points of generate.py's --anchors; compute_metrics.py's find_exit lists the fragment
 *              atoms bonded to linker atoms) judges where the linker bonds to the fragments:
 *     graph      the atoms and bonds of DL_CHECK_RINGS: checked atoms are rows with node_mask != 0, minus the pocket rows
 *                when drop_pocket applies; two atoms are bonded when dl_bond_orders gives an order > 0, decided over all of
 *                the molecule's checked atoms (the same n, so the n <= 25 and n > 25 forms switch where they do for the other
 *                bits), the pair oriented by the compacted atom order.
 *     roles      linker atoms: checked atoms with linker_mask != 0 (in the recovery rounds, the sub-batch's linker_mask, as
 *                DL_CHECK_NOVEL reads it); fragment atoms: the other checked atoms; anchors: fragment atoms whose anchor flag
 *                (dl_set_anchors, or dl_anchor_check's argument) is non-zero. Flags on linker rows, pocket rows and rows
 *                that are not checked are ignored.
 *     attachments  a_i of a fragment atom i: the number of bonds between i and a linker atom.
 *              DL_CHECK_ANCHORS holds iff a_i == 1 for every anchor and a_i == 0 for every other fragment atom: the linker
 *              attaches by exactly one bond at each anchor and nowhere else -- find_exit's list, repeats included, equals
 *              the anchor set. A molecule with no anchor passes (nothing was asked of it).
 *              Limits: these are dl_bond_orders' bonds, not OpenBabel's. An anchor that takes two linker bonds (a fused or
 *              spiro attachment) fails by design: the training data attaches one linker bond per anchor. A pair with a NaN
 *              coordinate compares false, so it is not bonded, as in the other checks.
 *              The check runs in a launch of its own (k_anchor_check) right after the check launch, before the
 *              DL_CHECK_UNIQUE verdict, which therefore sees the bit. dl_molecule_check and dl_novel_check refuse the bit;
 *              dl_anchor_check runs it on any batch.
 * dl_molecule_checks and dl_hash_sets do not grow for these: a positional initialiser of either struct fails -Wextra -Werror
 * once the struct gains a field, and existing C callers use such initialisers. The allowed sizes are engine state
 * (dl_set_ring_sizes) and the masks are read back with dl_last_ring_sizes; the anchor flags are per-call engine input
 * (dl_set_anchors).
 */
enum { DL_CHECK_CONNECTED = 1, DL_CHECK_VALENCE = 2, DL_CHECK_CLASH = 4, DL_CHECK_UNIQUE = 8, DL_CHECK_NOVEL = 16,
       DL_CHECK_RINGS = 32, DL_CHECK_ANCHORS = 64 };
typedef struct dl_molecule_checks {
  int32_t require;             /* OR of DL_CHECK_*, at least one: which verdicts make a row fail and be resampled */
  int32_t n_types;             /* columns of h that hold the atom type */
  const float* thr1;           /* (n_types,n_types) fp32 DEVICE, as dl_bond_orders; needed unless DL_CHECK_CLASH alone */
  const float* thr2;           /* needed for DL_CHECK_VALENCE, DL_CHECK_UNIQUE and DL_CHECK_NOVEL only */
  const float* thr3;
  const int32_t* max_valence;  /* (n_types) int32 DEVICE; DL_CHECK_VALENCE only */
  const float* clash;          /* (n_types,n_types) fp32 DEVICE, in pm, [min type][max type]; DL_CHECK_CLASH only */
} dl_molecule_checks;
/*
 * The hash sets of dl_sample_chain_retry_sets. DEVICE buffers, each in ascending unsigned order (duplicates allowed), read
 * while the call runs. A count of 0 is an empty set, whatever the pointer. It is a struct of its own rather than more fields
 * of dl_molecule_checks, so that existing positional initialisers of that struct still compile warning-free.
 */
typedef struct dl_hash_sets {
  const uint64_t* known;       /* (n_known): the known linker hashes of DL_CHECK_NOVEL; read with DL_CHECK_NOVEL only */
  int64_t n_known;
  const uint64_t* seen;        /* (n_seen): hashes that count as keepers in the DL_CHECK_UNIQUE verdict; read with
                                  DL_CHECK_UNIQUE only */
  int64_t n_seen;
} dl_hash_sets;
/*
 * Linker sizes drawn from a molecule's seed (no reference API; generate.py:88-99 draws them from one batch-level
 * Categorical.sample). Molecule b's size distribution is a table sizes[0..C) of ints >= 0 with finite fp32 logits
 * l_b[0..C): a SizeClassifier's output with sizes = its linker_id2size, all-zero logits over lo..hi for a uniform range, or
 * the one-entry table [n]. The draw with seed s:
 *   1. u = dl_size_uniform(s), a uniform in [0, 1) with 53 bits (below; a function of s alone, of no Philox draw);
 *   2. in fp64 and in index order: m = max_i l_i, e_i = exp(l_i - m), S = sum_i e_i, c_i = e_0 + ... + e_i;
 *   3. the drawn index is the first i with u * S < c_i, or, if rounding leaves none, the last i with e_i > 0; the size is
 *      sizes[i].
 * Attempt 0 uses the molecule's seed; recovery round a uses dl_retry_seed(seed, a), the seed of that round's noise, so the
 * seed that produced a row (seeds_used) determines both its size and its chain. A SizeClassifier mean-pools over the padded
 * rows of its input, so its logits -- and the size -- depend on the padding of the input batch: a molecule replays alone
 * with its seed only when its input is padded to the same number of rows.
 */
/*
 * dl_size_uniform(seed): the 53-bit uniform of the draw above. With the domain tag TAG = 0x6C696E6B65722D6E ("linker-n"):
 *     z = seed ^ TAG;  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;  z = (z ^ (z >> 27)) * 0x94D049BB133111EB;
 *     z = z ^ (z >> 31);  return (double)(z >> 11) * 2^-53;                      (all modulo 2^64)
 * A pure host function.
 */
double dl_size_uniform(uint64_t seed);
/*
 * The draw above for B molecules, without an engine. DEVICE buffers, enqueued on `stream`.
 *   logits     (B, logits_row_stride) fp32: molecule b's C logits from column 0; logits_row_stride >= C >= 1
 *   sizes      (C) int32: the size table
 *   seeds      (B) uint64: molecule b draws with dl_retry_seed(seeds[b], attempt) (attempt 0: seeds[b] itself)
 *   out_sizes  (B) int32 out
 */
dl_status dl_size_draw(int32_t B, int32_t C, const float* logits, int32_t logits_row_stride, const int32_t* sizes,
                       const uint64_t* seeds, int32_t attempt, int32_t* out_sizes, void* stream);
/*
 * What dl_sample_chain_retry redraws sizes from. DEVICE buffers, read while the call runs.
 */
typedef struct dl_size_redraw {
  int32_t C;                   /* entries of the size table, >= 1 */
  int32_t logits_row_stride;   /* >= C */
  const float* logits;         /* (B, logits_row_stride) fp32: molecule b's C logits */
  const int32_t* sizes;        /* (C) int32 >= 0: the size table */
  const int32_t* n_frag;       /* (B) int32: molecule b's fragment rows, pocket rows included, which come first */
  const float* linker_x;       /* (B, 3) fp32: the (normalised) coordinates of molecule b's template linker rows, the
                                  negated centre of mass of its template; given per molecule because a size-0 row has
                                  no linker row to copy them from */
} dl_size_redraw;
/*
 * dl_sample_chain_seeded that resamples only the molecules that fail: those that diverged and, with `checks`, those that
 * miss a required check. BLOCKING, unlike the other sampling entries: it runs the seeded loop and the checks (one launch),
 * synchronises `stream` once and reads the B flags and verdicts; then, for up to max_retries rounds, it gathers the failing
 * molecules into a sub-batch (B' molecules, same N), samples it with dl_retry_seed(seeds[b], a) in round a, checks it, and
 * writes the rows it takes back over those molecules' rows of every one of the keep_frames frames of `chain`, of nan_flags
 * and of passed. A row fails if its NaN flag is set or a required bit is missing; a resampled row replaces the caller's row
 * unless the caller's row is finite and the resample diverged. Rows that did not fail are not touched. Molecule b's row is
 * then what dl_sample_chain_seeded gives it alone with seed seeds_used[b] -- bit for bit on the SIMT edge path; on the
 * tensor-core path while no node tile rescales its fp16 operands, and a sub-batch of diverging molecules is where that
 * happens (DESIGN.md section 6). Both samplers, every graph type; cut-off graphs never read edge_mask, so the sub-batch gets
 * none.
 *   max_retries  >= 0 rounds (0: the seeded loop, the checks and the synchronisation: it only reports)
 *   nan_flags    (B) int32 DEVICE out, required: after the last round only the rows that still diverge are set
 *   seeds_used   (B) uint64 DEVICE out: the seed that produced each returned row (its attempt's dl_retry_seed)
 *   attempts     (B) int32 DEVICE out: the attempt that produced each row, 0 = the first draw
 *   checks       the molecule checks (dl_molecule_checks), or NULL: NaN recovery alone, and `passed` is not read.
 *                1 <= n_types <= in_node_nf, N <= 8192. DL_CHECK_CLASH reads the linker rows of linker_mask (of the
 *                sub-batch in the rounds) and checks->clash; it is DL_ERR_INVALID without a table, on DL_GRAPH_FC (no pocket
 *                rows) and with DL_SAMPLER_INPAINT (whose loop re-noises the pocket).
 *   passed       (B) int32 DEVICE out, required with `checks`: the OR of the DL_CHECK_* bits row b's returned molecule
 *                satisfies, among those required. DL_CHECK_UNIQUE (needs thr1, thr2 and thr3) is the verdict stated at
 *                DL_CHECK_UNIQUE above, over the rows of this call: it runs after the first loop's checks and after every
 *                round's, on the device. Without it there is no extra launch or allocation; with it the full batch's hashes
 *                live in the engine (cached by B), not in a caller buffer. DL_CHECK_NOVEL (needs thr1, thr2 and thr3) reads
 *                the linker rows of linker_mask (of the sub-batch in the rounds) and hashes them in the same launch as the
 *                other checks; through this entry its known set is empty, so every row passes it (the set is an argument
 *                of dl_sample_chain_retry_sets). DL_CHECK_RINGS (needs thr1) reads the linker rows of linker_mask (of the
 *                sub-batch in the rounds) and the allowed sizes of dl_set_ring_sizes, and is DL_ERR_INVALID before that
 *                has been called on the engine; dl_last_ring_sizes returns the masks. DL_CHECK_ANCHORS (needs thr1) reads
 *                the linker rows of linker_mask (of the sub-batch in the rounds) and the anchor flags of dl_set_anchors (of
 *                the caller's row, row for row, in the rounds), and is DL_ERR_INVALID unless dl_set_anchors was called with
 *                this B and N since the engine's previous dl_sample_chain_retry(_sets) call. Without it there is no extra
 *                launch or allocation. Bits 128 and up are refused.
 *   redraw       the sizes to redraw each resampled row's linker size from (dl_size_redraw), or NULL: sizes stay fixed,
 *                and `sizes_used` is not read
 *   sizes_used   (B) int32 DEVICE in/out, required with `redraw`: the attempt-0 sizes on entry; on return, the size of every
 *                returned row (a row that is not taken keeps its size)
 * Rows that merely miss a check after the last round are valid samples: they are returned with their bits cleared and do not
 * make the call fail. Returns DL_NAN_DETECTED only if some row still diverges after the last round. A row whose fragments
 * alone break the valence rule cannot be repaired by a new linker: it is resampled every round and comes back with the bit
 * cleared (vet inputs with dl_molecule_check).
 * With `redraw`, the inputs are the template of the attempt-0 sizes (dl_size_draw with attempt 0) padded to the capacity
 * N >= max_b n_frag[b] + max(sizes), which every redrawn size fits. In round a, each failing row b draws size s' with
 * dl_retry_seed(seeds[b], a) and is gathered as the template of that size:
 *   rows [0, n_frag[b])                copied from the inputs;
 *   rows [n_frag[b], n_frag[b] + s')   linker rows: node_mask 1, linker_mask 1, fragment_mask 0, x = linker_x[b], h 0,
 *                                      context 0;
 *   later rows                          zero; on DL_GRAPH_FC the edge-mask block is batching's int8 rule over the live rows
 *                                      (-1 off the diagonal, -2 on it, 0 elsewhere).
 * It is DL_ERR_INVALID with DL_SAMPLER_INPAINT (which has no linker size) and when N < n_frag[b] + max(sizes) for some b.
 * Row b's size and chain are then those molecule b gets alone, padded to N, with seed seeds_used[b] -- subject to the padding
 * rule of the size draw above and to the tensor-core caveat above.
 * The sub-batch has a workspace of its own, cached by (B', N); the full batch's is neither freed nor resized.
 * dl_last_elapsed_ms keeps timing the first loop.
 */
dl_status dl_sample_chain_retry(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                                const float* xh, const int8_t* node_mask, const float* fragment_mask, const float* linker_mask,
                                const int8_t* edge_mask, const float* context, const uint64_t* seeds, const dl_step_coef* coef,
                                const float* norm, float* chain, int32_t* nan_flags, int32_t max_retries, uint64_t* seeds_used,
                                int32_t* attempts, const dl_molecule_checks* checks, int32_t* passed,
                                const dl_size_redraw* redraw, int32_t* sizes_used, void* stream);
/*
 * dl_sample_chain_retry with the hash sets of DL_CHECK_NOVEL and DL_CHECK_UNIQUE (dl_hash_sets): `known` is the set
 * DL_CHECK_NOVEL tests each row's linker hash against, `seen` the hashes that count as keepers in the DL_CHECK_UNIQUE
 * verdict. sets == NULL, or both counts 0, is dl_sample_chain_retry itself: no extra launch. Before the first loop it
 * checks, on `stream`, that every set in use (known with DL_CHECK_NOVEL, seen with DL_CHECK_UNIQUE, count > 0) is in
 * ascending unsigned order; a set that is not, a pointer that is not device or managed memory of the engine's device, a NULL
 * pointer with a positive count, a negative count or sets without `checks` is DL_ERR_INVALID.
 *   linker_hashes  (B) uint64 DEVICE out or NULL; needs DL_CHECK_NOVEL: the linker hash L the check computed for every
 *                  returned row -- the L its DL_CHECK_NOVEL bit was decided on.
 * Everything else is dl_sample_chain_retry's.
 */
dl_status dl_sample_chain_retry_sets(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                                     const float* xh, const int8_t* node_mask, const float* fragment_mask,
                                     const float* linker_mask, const int8_t* edge_mask, const float* context,
                                     const uint64_t* seeds, const dl_step_coef* coef, const float* norm, float* chain,
                                     int32_t* nan_flags, int32_t max_retries, uint64_t* seeds_used, int32_t* attempts,
                                     const dl_molecule_checks* checks, const dl_hash_sets* sets, int32_t* passed,
                                     uint64_t* linker_hashes, const dl_size_redraw* redraw, int32_t* sizes_used,
                                     void* stream);
/*
 * The checks alone, on any (B,N) batch. DEVICE buffers, enqueued on `stream`.
 *   xh        (B,N,>=3+n_types) fp32, row stride xh_row_stride: x at columns 0..2, the atom-type one-hot from column 3
 *   node_mask (B,N) int8
 *   context   (B,N,context_nf) fp32; with drop_pocket != 0 the rows whose column context_nf - 1 is non-zero are not atoms
 *             (read only then; may be NULL otherwise)
 *   passed    (B) int32 out, as above
 *   valence   (B,N) int32 out or NULL; needs DL_CHECK_VALENCE: each checked atom's valence, 0 on every other row (for a
 *             hand-off to RDKit, and for tests)
 * 1 <= N <= 8192. require takes DL_CHECK_CONNECTED and DL_CHECK_VALENCE only; the clash check alone is dl_clash_check, and
 * DL_CHECK_UNIQUE, a verdict on molecules compared with each other, has no per-molecule form: dl_molecule_hash gives the
 * hashes it compares. DL_CHECK_NOVEL needs a linker_mask, which this entry does not take: the linker hashes are
 * dl_molecule_hash over node_mask AND linker_mask. DL_CHECK_RINGS runs through dl_ring_check and DL_CHECK_ANCHORS through
 * dl_anchor_check.
 */
dl_status dl_molecule_check(int32_t B, int32_t N, const dl_molecule_checks* checks, const float* xh, int32_t xh_row_stride,
                            const int8_t* node_mask, const float* context, int32_t context_nf, int32_t drop_pocket,
                            int32_t* passed, int32_t* valence, void* stream);
/*
 * The checks with DL_CHECK_NOVEL, on any (B,N) batch, without an engine: the check launch of dl_sample_chain_retry_sets.
 * DEVICE buffers, enqueued on `stream` of the current device.
 *   checks       require includes DL_CHECK_NOVEL and may add DL_CHECK_CONNECTED, DL_CHECK_VALENCE, DL_CHECK_CLASH (needs
 *                checks->clash and drop_pocket) and DL_CHECK_UNIQUE (needs `hash`; the bit itself is a verdict over a
 *                call's rows and stays clear). Tables as for dl_sample_chain_retry. DL_CHECK_RINGS runs through
 *                dl_ring_check and DL_CHECK_ANCHORS through dl_anchor_check.
 *   sets         known (ascending unsigned order, not checked here) or NULL: an empty set; seen is not read
 *   xh, node_mask, context, context_nf, drop_pocket   as dl_molecule_check
 *   linker_mask  (B,N) fp32: the checked rows with linker_mask != 0 are the linker atoms
 *   passed       (B) int32 out: the bits of require the molecule satisfies (DL_CHECK_UNIQUE clear)
 *   linker_hash  (B) uint64 out or NULL: molecule b's L
 *   hash         (B) uint64 out, with DL_CHECK_UNIQUE: molecule b's H
 * 1 <= n_types <= xh_row_stride - 3, 1 <= N <= 8192.
 */
dl_status dl_novel_check(int32_t B, int32_t N, const dl_molecule_checks* checks, const dl_hash_sets* sets, const float* xh,
                         int32_t xh_row_stride, const int8_t* node_mask, const float* linker_mask, const float* context,
                         int32_t context_nf, int32_t drop_pocket, int32_t* passed, uint64_t* linker_hash, uint64_t* hash,
                         void* stream);
/*
 * DL_CHECK_CLASH alone, on any (B,N) batch, without an engine. DEVICE buffers, enqueued on `stream`.
 *   clash       (n_types,n_types) fp32, in pm, as dl_molecule_checks.clash
 *   xh          (B,N,>=3+n_types) fp32, row stride xh_row_stride, as dl_molecule_check
 *   node_mask   (B,N) int8
 *   linker_mask (B,N) fp32: the rows checked against the pocket (to vet a fragment, pass the fragment rows here)
 *   context     (B,N,context_nf) fp32, context_nf >= 1: column context_nf - 1 marks the pocket rows
 *   passed      (B) int32 out: DL_CHECK_CLASH or 0
 *   clashes     (B,N) int32 out or NULL: for each linker atom, the number of pocket atoms it clashes with; 0 on every
 *               other row
 * 1 <= n_types <= xh_row_stride - 3, 1 <= N <= 8192.
 */
dl_status dl_clash_check(int32_t B, int32_t N, int32_t n_types, const float* clash, const float* xh, int32_t xh_row_stride,
                         const int8_t* node_mask, const float* linker_mask, const float* context, int32_t context_nf,
                         int32_t* passed, int32_t* clashes, void* stream);
/*
 * One clash-guidance push (stated at dl_set_clash_guidance) on any (B,N) batch, without an engine. DEVICE buffers, enqueued
 * on `stream`.
 *   clash       (n_types,n_types) fp32, in pm, as dl_molecule_checks.clash: r_ik = clash[min type][max type] / 100 Angstrom;
 *               a negative entry exempts the pair
 *   scale       lambda, finite and >= 0 (0: nothing is launched)
 *   xh          (B,N,>=3+n_types) fp32 in/out, row stride xh_row_stride: x at columns 0..2, the type channels from column 3
 *               (an atom's type is the first maximum of its first n_types channels). Only columns 0..2 of linker rows with a
 *               contributing pair are written.
 *   node_mask   (B,N) int8
 *   linker_mask (B,N) fp32
 *   context     (B,N,context_nf) fp32, context_nf >= 1: column context_nf - 1 marks the pocket rows
 * The rows are dl_clash_check's. 1 <= n_types <= xh_row_stride - 3, 1 <= N <= 8192.
 */
dl_status dl_clash_guide(int32_t B, int32_t N, int32_t n_types, const float* clash, float scale, float* xh,
                         int32_t xh_row_stride, const int8_t* node_mask, const float* linker_mask, const float* context,
                         int32_t context_nf, void* stream);
/*
 * The graph hash of DL_CHECK_UNIQUE alone, on any (B,N) batch, without an engine. DEVICE buffers, enqueued on `stream`.
 *   checks    n_types, thr1, thr2 and thr3 are read; require, max_valence and clash are not
 *   xh, node_mask, context, context_nf, drop_pocket   as dl_molecule_check: the atoms and types of dl_molecule_checks
 *   hash      (B) uint64 out: molecule b's H
 * 1 <= n_types <= xh_row_stride - 3, 1 <= N <= 8192.
 */
dl_status dl_molecule_hash(int32_t B, int32_t N, const dl_molecule_checks* checks, const float* xh, int32_t xh_row_stride,
                           const int8_t* node_mask, const float* context, int32_t context_nf, int32_t drop_pocket,
                           uint64_t* hash, void* stream);
/*
 * DL_CHECK_RINGS alone, on any (B,N) batch, without an engine. DEVICE buffers, enqueued on `stream`.
 *   thr1        (n_types,n_types) fp32, as dl_molecule_checks.thr1: the bonds
 *   xh, node_mask, context, context_nf, drop_pocket   as dl_molecule_check: the checked atoms
 *   linker_mask (B,N) fp32: the checked rows with linker_mask != 0 are the linker atoms
 *   allowed     the ring sizes that pass (bits 0-2 clear), as dl_set_ring_sizes
 *   passed      (B) int32 out: DL_CHECK_RINGS or 0
 *   ring_sizes  (B) uint64 out or NULL: molecule b's ring-size mask
 * 1 <= n_types <= xh_row_stride - 3, 1 <= N <= 8192. It judges DL_CHECK_RINGS alone: DL_CHECK_ANCHORS is dl_anchor_check.
 */
dl_status dl_ring_check(int32_t B, int32_t N, int32_t n_types, const float* thr1, const float* xh, int32_t xh_row_stride,
                        const int8_t* node_mask, const float* linker_mask, const float* context, int32_t context_nf,
                        int32_t drop_pocket, uint64_t allowed, int32_t* passed, uint64_t* ring_sizes, void* stream);
/*
 * The ring sizes DL_CHECK_RINGS allows in the following dl_sample_chain_retry(_sets) calls: bit k set lets a smallest ring
 * of k atoms pass, bit 63 one of 63 or more (stated at DL_CHECK_RINGS). Sticky like dl_set_start_step; read only by calls
 * whose checks require the bit. DL_ERR_INVALID: bits 0-2 set.
 */
dl_status dl_set_ring_sizes(dl_engine* e, uint64_t allowed);
/*
 * The ring-size mask of every returned row of the engine's last dl_sample_chain_retry(_sets) call -- the mask its
 * DL_CHECK_RINGS bit was decided on -- copied to out, (B) uint64 DEVICE, on `stream`. DL_ERR_INVALID when that call did not
 * require DL_CHECK_RINGS (or failed before returning rows), or had another B.
 */
dl_status dl_last_ring_sizes(dl_engine* e, int32_t B, uint64_t* out, void* stream);
/*
 * DL_CHECK_ANCHORS alone, on any (B,N) batch, without an engine. DEVICE buffers, enqueued on `stream`.
 *   thr1        (n_types,n_types) fp32, as dl_molecule_checks.thr1: the bonds
 *   xh, node_mask, context, context_nf, drop_pocket   as dl_molecule_check: the checked atoms
 *   linker_mask (B,N) fp32: the checked rows with linker_mask != 0 are the linker atoms
 *   anchors     (B,N) int8: the anchor flags (stated at DL_CHECK_ANCHORS)
 *   passed      (B) int32 out: DL_CHECK_ANCHORS or 0
 *   attachments (B,N) int32 out or NULL: a_i on every fragment atom, 0 on every other row
 * 1 <= n_types <= xh_row_stride - 3, 1 <= N <= 8192.
 */
dl_status dl_anchor_check(int32_t B, int32_t N, int32_t n_types, const float* thr1, const float* xh, int32_t xh_row_stride,
                          const int8_t* node_mask, const float* linker_mask, const int8_t* anchors, const float* context,
                          int32_t context_nf, int32_t drop_pocket, int32_t* passed, int32_t* attachments, void* stream);
/*
 * The anchor flags of the engine's next dl_sample_chain_retry(_sets) call: (B,N) int8 (host or DEVICE), row b's flags
 * those of molecule b (stated at DL_CHECK_ANCHORS). Copied into an engine buffer, cached by (B,N), on `stream`. Not sticky:
 * the next dl_sample_chain_retry(_sets) call on the engine reads the flags and clears them, whether or not its checks
 * require DL_CHECK_ANCHORS, so per-row data never carries over to a later batch. DL_ERR_INVALID: B or N < 1, NULL anchors.
 */
dl_status dl_set_anchors(dl_engine* e, int32_t B, int32_t N, const int8_t* anchors, void* stream);
/* Device time (ms, CUDA events) of the retry rounds of the most recent dl_sample_chain_retry, each from its row gather to
 * its row scatter -- including the wait for the host to capture the sub-batch's step graph -- summed over the rounds; 0 when
 * no round ran. */
float dl_last_retry_ms(dl_engine* e);
/* Strong scaling (SURVEY 8(e)): this engine samples molecules [b0, b0 + B) of a batch of B_full. The device-side noise of
 * the following dl_sample_chain_rng / dl_noise_fill / dl_noise_fill_inpaint calls is then the slice's ROWS of the
 * full-batch draws (and offset_consumed is the full batch's), so the gathered result is bit-identical to the single-GPU
 * run whatever the split -- on the SIMT path, and on the tensor-core path while no sample diverges far enough for the node
 * GEMM to rescale a tile's fp16 operands (tiles span molecules, so the split moves them; DESIGN.md section 6). B_full = 0
 * switches it off. */
dl_status dl_set_noise_slice(dl_engine* e, int32_t B_full, int32_t b0);
/*
 * Partial diffusion (no reference API; the `optimize` mode of DiffSBDD): the following dl_sample_chain* calls of this engine,
 * the recovery rounds of dl_sample_chain_retry included, vary the linker the caller's xh holds on its linker_mask rows
 * instead of sampling one from pure noise. With 0 <= t0 <= T:
 *   z     = xh * fragment_mask + (alpha_t0 * xh + sigma_t0 * eps) * linker_mask,   eps = draw 0 * linker_mask
 *           -- q(z_t0 | x) as EDM.forward draws it (edm.py:67-74), each product and sum rounded on its own; alpha_t0 and
 *           sigma_t0 are sqrt(sigmoid(-gamma)) and sqrt(sigmoid(gamma)) of gamma(t0 / T), evaluated as the caller evaluates
 *           the coefficient table;
 *   steps s = t0-1 .. 0 with rows T-1-s of `coef` (time feature (s+1)/T), then the final step with row T.
 * The draws are eps, one per step and the final draw: t0 + 2, in the order of dl_sample_chain_rng -- a noise tensor holds t0 + 2
 * slabs, offset_consumed is (t0 + 2) * per_draw, and a per-molecule stream uses its draws 0 .. t0+1. Frames with no step
 * below t0 stay zero; chain[0] is the final sample. The NaN flags' row tag counts the loop's rows from the start step: row
 * j is step t0-1-j. t0 = T is not the plain sampler: z_T keeps alpha_T * xh. DL_SAMPLER_INPAINT with a start step set, or
 * t0 > T, is DL_ERR_INVALID at the sampling call. A negative t0 clears the start step (the default). Non-finite alpha_t0 or
 * sigma_t0 is DL_ERR_INVALID.
 */
dl_status dl_set_start_step(dl_engine* e, int32_t t0, float alpha_t0, float sigma_t0);
/*
 * Partial diffusion from per-molecule start steps (no reference API): with host arrays t0, alpha and sigma of B entries,
 * 0 <= t0[b] <= T, molecule b of the following sampling calls of this engine -- the recovery rounds included -- is sampled
 * exactly as dl_set_start_step(t0[b], alpha[b], sigma[b]) samples it, whatever the other rows' steps:
 *   start  z_b = xh * fragment_mask + (alpha[b] * xh + sigma[b] * eps) * linker_mask; (alpha[b], sigma[b]) are the
 *          scalars of t0[b] the caller evaluates at the call's own B (EDM.start_scalars(t0[b], B)), since they depend on it;
 *   steps  t0[b]-1 .. 0 with rows T-1-s of `coef`, then the final row T;
 *   draws  row b's draw k is its own k-th draw: draw 0 is eps, step s consumes draw t0[b] - s and the final step draw
 *          t0[b] + 1. A noise tensor holds t0max + 2 slabs (t0max = max_b t0[b]) of which row b reads slabs 0 .. t0[b]+1
 *          of its own row; per-molecule seeds use their stream's draws 0 .. t0[b]+1;
 *   output frames with no step below t0[b] stay zero for row b; until row b starts, its z is held bit for bit; its NaN
 *          flag ignores every forward it is not part of, and its row tag counts from its own start: tag row j is step
 *          t0[b]-1-j.
 * Row b of a call thus equals row b of the single-step call with t0[b] on the same batch, seeds or noise rows: bit for bit
 * on the SIMT edge path, and on the tensor-core path within the per-molecule rule (node tiles span molecules, the caveat of
 * batch slices and sub-batches). With every t0[b] equal, the call is the dl_set_start_step call, bit for bit on both paths.
 * The engine orders the rows by t0 descending (stably), gathers their inputs in that order, and loop step r computes only
 * the prefix of rows that have started, recapturing the step graph when the prefix grows: a call costs
 * sum_b (t0[b] + 1) molecule-steps instead of B * (t0max + 1) (dl_last_molecule_steps).
 * B = 0 clears them. Setting either this or dl_set_start_step clears the other. DL_ERR_INVALID: here, a negative t0[b] or a
 * non-finite scalar; at the sampling call, a B other than the one set, t0[b] > T, DL_SAMPLER_INPAINT, dl_sample_chain_rng
 * (the batch stream's draws are not per row) and a dl_size_redraw (linker sizes take no start step).
 */
dl_status dl_set_start_steps(dl_engine* e, int32_t B, const int32_t* t0, const float* alpha, const float* sigma);
/*
 * RePaint resampling (Lugmayr et al., 2022; DiffSBDD's inpaint(..., resamplings=r); no reference API) for DL_SAMPLER_INPAINT:
 * with r >= 1, reverse step s = T-1 .. 0 of the following dl_sample_chain, _rng, _seeded, _retry and _retry_sets calls of
 * this engine -- the recovery rounds included -- becomes r passes. Pass u = 0 .. r-1:
 *   denoise   the plain inpainting step (row T-1-s of `coef`, time feature (s+1)/T on every pass): p(z_s | z_t) on all atoms,
 *             q(z_s | z_t, x) on the fragment atoms, combined by the masks and projected to a zero centre of mass;
 *   re-noise  for u < r-1: z <- alpha_t|s * z + sigma_t|s * eps on every atom, eps COM-free on the node mask (coordinates)
 *             and masked (features) like the p draw; each product and the sum rounded on its own. No projection follows:
 *             the next pass projects.
 * The frame of step s is written after its last pass; the final p(x, h | z_0) step is unchanged. `jump` holds (T, 2) HOST
 * floats, (alpha_t|s, sigma_t|s) of sigma_and_alpha_t_given_s(gamma_t, gamma_s) per row in dl_step_coef row order (row j is
 * step T-1-j). The draws are z_T; then per step and pass the p and q draws and, for u < r-1, the re-noise draw; then the two
 * final draws: 1 + T(3r-1) + 2 in that order, which a noise tensor holds as prepared slabs, offset_consumed counts and
 * dl_noise_fill_inpaint writes. The NaN flags' row tag names the step, whatever the pass. r = 1 (the default) restores
 * the plain loop, bit for bit and with the same launches. Sticky like dl_set_start_step. DL_ERR_INVALID: here, r < 1,
 * r > 1 with a null jump, T < 1 or a non-finite jump value; at the sampling call, with r > 1, a T other than the one set
 * and DL_SAMPLER_LINKER. A call costs about r times the plain loop (T*r + 1 forwards).
 */
dl_status dl_set_resamplings(dl_engine* e, int32_t r, int32_t T, const float* jump);
/*
 * Clash guidance (no reference API; a sampler tool that makes no claim about chemistry) for DL_SAMPLER_LINKER on cut-off
 * (pocket) graphs: in the following dl_sample_chain* calls of this engine -- the recovery rounds of dl_sample_chain_retry
 * included -- after the reverse update has produced z_s at a step s < steps, and before anything reads it, every molecule's
 * linker atoms are pushed away from its pocket atoms:
 *   p_i <- p_i + scale * sum_k max(0, r_ik - d_ik) (p_i - p_k) / d_ik,   d_ik = |p_i - p_k|
 * with p the coordinate columns of z_s, i over the linker atoms (node_mask, linker_mask != 0 and context column C - 1 == 0)
 * and k over the pocket atoms (node_mask and column C - 1 != 0): the rows of DL_CHECK_CLASH. r_ik = clash[min type][max
 * type] / 100 Angstrom of the (n_types,n_types) HOST table in pm; a negative entry exempts the pair. The table is copied
 * into host memory here, and each following sampling call uploads that copy on the engine's loop stream, ordered after
 * the calls enqueued before it: setting another table never changes a call already made, even one still running. An atom's
 * type is the first maximum of its first n_types feature channels in z_s. Every term is taken from the state before the
 * push; a pair at d_ik = 0 or with a NaN distance contributes nothing. Only the coordinates of linker rows change; the
 * final p(x, h | z_0) step is never guided. A frame written at a guided step holds the guided state, and the next step's
 * cut-off graph is built from it. Guidance draws no noise: draws and their count are unchanged. The sum over the pocket
 * atoms has a fixed shape and no atomics, so a molecule's result depends neither on its batch-mates nor on the launch.
 * One launch per step of the captured step graph decides on the device whether its step is guided.
 * Sticky like dl_set_start_step. steps = 0 or scale = 0 switches it off: the calls then launch exactly what they launch
 * without it. DL_ERR_INVALID: here, a non-finite or negative scale, steps < 0, and n_types < 1 or a NULL table while on; at
 * the sampling call, steps > T, DL_SAMPLER_INPAINT, a start step (dl_set_start_step or dl_set_start_steps), DL_GRAPH_FC,
 * n_types > F, N > 8192 and a NULL context.
 */
dl_status dl_set_clash_guidance(dl_engine* e, float scale, int32_t steps, int32_t n_types, const float* clash);
/*
 * ODE solvers for DL_SAMPLER_LINKER (no reference API): the following dl_sample_chain* calls of this engine -- the recovery
 * rounds of dl_sample_chain_retry included -- replace the ancestral update p(z_s | z_t) by a deterministic step of the
 * probability-flow ODE, so a sample is a function of its z_T (or its q(z_t0 | x)) alone. With alpha = sqrt(sigmoid(-gamma)),
 * sigma = sqrt(sigmoid(gamma)), lambda = -gamma / 2 at t = (s+1)/T and s/T, and h = lambda_s - lambda_t > 0, row r < T of
 * the (T + 1, 8) HOST fp32 `table` (step s = T-1-r, dl_step_coef's row order) holds
 *   [0] sigma_t   [1] 1/alpha_t   [2] sigma_s/sigma_t   [3] c1 = -alpha_s expm1(-h)
 *   [4] c2a = c1 (1 + 1/(2 rho))   [5] c2b = -c1 / (2 rho)   [6] h   [7] 0,      rho = h_{r-1} / h_r
 * and row T [0] sigma_0, [1] 1/alpha_0, the rest 0. EDM.solver_coefficients builds it, each entry evaluated in fp64 from the
 * fp32 gamma table and rounded once; for DL_SOLVER_DDIM, and in row 0, c2a = c1 and c2b = 0. On linker rows, eps = the
 * dynamics output times linker_mask and
 *   xhat = [1] * (z_t - [0] * eps)                         (the data prediction)
 *   z_s  = [2] * z_t + [3] * xhat                          (DDIM; DPM-Solver++(2M) at a row's first step)
 *   z_s  = [2] * z_t + ([4] * xhat + [5] * xhat')          (DPM-Solver++(2M) after it; xhat' = the row's previous xhat)
 *   final row: x = xhat, with no sigma_x noise, then unnormalised and one-hot as the ancestral sampler's final row.
 * Fragment rows keep z_t bit for bit and padded rows stay 0, as in the ancestral loop. A row's first step is the loop's
 * first (its start step with dl_set_start_step), or its own start step with dl_set_start_steps; a recovery round starts its
 * rows afresh. The history lives in the engine's workspace. The draws are those of the ancestral loop, in count and order
 * (T + 2, or t0 + 2), so the device streams advance as they do without a solver, but only draw 0 (z_T, or the eps of
 * q(z_t0 | x)) is read. dl_step_coef keeps giving the time feature and the frames. Clash guidance (dl_set_clash_guidance)
 * pushes z_s after the update and never the history.
 * The table is copied into host memory here, and each following call uploads the rows it runs on the engine's loop stream,
 * so a call already enqueued keeps its table. Sticky like dl_set_resamplings. kind = DL_SOLVER_ANCESTRAL switches it off
 * (T and table are ignored): the calls then launch exactly what they launch without it. DL_ERR_INVALID: here, an unknown
 * kind, and while on a NULL table, T outside [1, 2^24], a non-finite entry or a row r < T with h <= 0; at the sampling
 * call, a T other than the one set and DL_SAMPLER_INPAINT.
 */
dl_status dl_set_solver(dl_engine* e, int32_t kind, int32_t T, const float* table);
/*
 * Fixed atoms for DL_SAMPLER_LINKER (scaffold-constrained generation by replacement, as RePaint replaces known pixels; no
 * reference API): the engine's next dl_sample_chain* call -- and the recovery rounds of a dl_sample_chain_retry(_sets) call
 * -- keeps the linker rows whose (B, N) int8 DEVICE flag `fixed` is non-zero at the coordinates and types of the call's
 * xh, and samples the other linker rows around them. The kept rows stay noisy linker rows throughout, as the linker
 * denoiser was trained to see them: with xh the row's normalised input, eps_0 its own draw 0, and (alpha_s, sigma_s) row
 * r = T-1-s of the (T + 1, 2) HOST fp32 `scalars` (dl_step_coef's row order; row T holds (alpha_T, sigma_T)),
 *   start                   alpha xh + sigma eps_0, as the partial-diffusion start forms it (k_init_z_rows), with the
 *                           scalars of the call's start: row T from noise, dl_set_start_step's, or each row's own
 *                           dl_set_start_steps scalars
 *   step s < T, ancestral   alpha_s xh + sigma_s nz_s, nz_s the draw the update reads for the row and would otherwise
 *                           scale by sigma; the draws stay those of the plain call in count and order, so seeds, offsets
 *                           and noise tensors mean what they mean without this call
 *   step s < T, dl_set_solver  alpha_s xh + sigma_s eps_0 (the probability-flow path of a known point); the 2M history of
 *                           a kept row never enters it
 *   final step              xh, so chain[0] holds the input's x times norm[0] (bit for bit when norm[0] is a power of two,
 *                           as for every DiffLinker model) and the one-hot of its types
 * Each product and the sum is rounded on its own. Frames hold the replaced state, unnormalised like every row. The network
 * sees the kept rows as linker rows, and the molecule checks count them as linker atoms. Clash guidance
 * (dl_set_clash_guidance) neither moves the kept rows nor lets them push. EDM.fixed_atom_scalars builds `scalars` as
 * start_scalars(s, B) row by row (q(z_s | x)'s alpha and sigma as EDM.forward evaluates them at the call's batch size).
 * Per-call input like dl_set_anchors: the flags are copied on `stream` (the call reads them while its loop runs), the
 * scalars into host memory, uploaded on the loop stream by the call; every dl_sample_chain* call reads and clears the
 * setting, whether or not it uses it. fixed = NULL switches it off (the other arguments are ignored): the calls then launch
 * exactly what they launch without it. DL_ERR_INVALID: here, B or N < 1, T outside [1, 2^24], NULL scalars or a
 * non-finite one; at the sampling call, which then blocks once to vet the flags, a B, N or T other than the ones set,
 * DL_SAMPLER_INPAINT, a size redraw (dl_size_redraw), a flag on a row that is not a live linker row (node_mask and
 * linker_mask non-zero, fragment_mask 0: fragment, pocket and padding rows), and a flagged row whose type channels are not
 * a normalised one-hot (one channel (1 - norm[2]) / norm[1], the others (0 - norm[2]) / norm[1], in fp32).
 */
dl_status dl_set_fixed_atoms(dl_engine* e, int32_t B, int32_t N, const int8_t* fixed, int32_t T, const float* scalars,
                             void* stream);
/*
 * Linker types for DL_SAMPLER_LINKER (no reference API): the engine's next dl_sample_chain* call -- and the recovery rounds
 * of a dl_sample_chain_retry(_sets) call, each row with its molecule's mask -- gives every linker atom of molecule b a type
 * that bit c of the HOST mask masks[b] allows (type channel c, c < F). On every free linker row (linker_mask non-zero, not
 * kept by dl_set_fixed_atoms) each step constrains the data prediction of the excluded channels to the one-hot's
 * normalised off value, off = (0 - norm[2]) / norm[1]:
 *   ancestral update        eps_c = (z_t,c - alpha_t off) / sigma_t, which gives xhat_c = (z_t,c - sigma_t eps_c) / alpha_t
 *                           = off; (alpha_t, sigma_t) is row t - 1 of the (T + 1, 2) HOST fp32 `scalars` at a step from
 *                           t >= 1 (dl_step_coef's row order, so row r holds step s = T-1-r), and row T at the step from T
 *   dl_set_solver           xhat_c = off, which also enters the DPM-Solver++(2M) history
 *   final step              the one-hot of chain[0] takes the argmax over the allowed channels only
 * so every linker atom of chain[0] has an allowed type by construction. Kept rows and fragment and pocket rows are not
 * changed. No draw is added or moved, so seeds, offsets and noise tensors mean what they mean without this call.
 * Intermediate frames (keep_frames > 1) hold continuous states, which carry no such guarantee. EDM.fixed_atom_scalars builds
 * `scalars`. Per-call input like dl_set_anchors: masks and scalars are copied into host memory here and uploaded on the loop
 * stream by the call; every dl_sample_chain* call reads and clears the setting, whether or not it uses it. masks = NULL
 * switches it off (the other arguments are ignored): the calls then launch exactly what they launch without it.
 * DL_ERR_INVALID: here, B < 1, F other than dl_config.in_node_nf, a mask of 0 or with bits at or above F, T outside
 * [1, 2^24], NULL scalars or a non-finite one; at the sampling call, a B or T other than the ones set, DL_SAMPLER_INPAINT,
 * and, with dl_set_fixed_atoms, a kept row whose one-hot type its molecule's mask excludes (vetted in the blocking check
 * of dl_set_fixed_atoms).
 */
dl_status dl_set_linker_types(dl_engine* e, int32_t B, int32_t F, const uint32_t* masks, int32_t T, const float* scalars);
/* The (n_draws,B,N,3+F) tensor the device-side stream of dl_sample_chain_rng stands for (tests, debugging). DEVICE out. */
dl_status dl_noise_fill(dl_engine* e, int32_t n_draws, int32_t B, int32_t N, uint64_t seed, uint64_t offset, float* out,
                        uint64_t* offset_consumed, void* stream);
/* The (2T+3,B,N,3+F) prepared draws the device-side stream of dl_sample_chain_rng(DL_SAMPLER_INPAINT) stands for, computed by
 * the same device code (tests, debugging); with r resampling passes set (dl_set_resamplings), the 1 + T(3r-1) + 2 draws of
 * that loop. node_mask (B,N) int8, fragment_mask (B,N) fp32, out: DEVICE. */
dl_status dl_noise_fill_inpaint(dl_engine* e, int32_t T, int32_t B, int32_t N, const int8_t* node_mask,
                                const float* fragment_mask, uint64_t seed, uint64_t offset, float* out,
                                uint64_t* offset_consumed, void* stream);

/* HOST-buffer variant of dl_sample_chain (pinned or pageable): H2D of all inputs incl. noise, loop, D2H of chain and flags,
 * synchronises. Returns DL_NAN_DETECTED if any flag is set. */
dl_status dl_sample_chain_host(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                               const float* xh, const int8_t* node_mask, const float* fragment_mask,
                               const float* linker_mask, const int8_t* edge_mask, const float* context,
                               const float* noise, const dl_step_coef* coef, const float* norm, float* chain,
                               int32_t* nan_flags);

/* Instrumentation for bench.py: kernels launched by this engine since creation, and the device time (ms)
 * of the most recent dl_sample_chain loop / dl_dynamics_forward measured with CUDA events on `stream`
 * (valid after the stream has been synchronised). */
int64_t dl_launch_count(const dl_engine* e);
/* The molecule-steps the most recent sampling loop computed, summed over its steps: B * (t0 + 1) with one start step
 * (B * (T + 1) without), sum_b (t0[b] + 1) with per-molecule ones, B * (T * r + 1) with r resampling passes (every pass
 * counts). The recovery rounds keep the first loop's. */
int64_t dl_last_molecule_steps(dl_engine* e);
float dl_last_elapsed_ms(dl_engine* e);
/* Average device time (ms, CUDA events on the engine's loop stream) of the dominant kernel -- the layer-0 GCL
 * edge kernel -- relaunched `reps` times on the engine's current workspace (state of the last call; the
 * caller's mask tensors of that call must still be alive). Blocking. Negative on error. For bench.py's roofline. */
float dl_time_edge_kernel(dl_engine* e, int32_t reps);
/* Cut-off (pocket) graphs, tensor-core path: what the neighbour-list kernel packed for the most recent forward call --
 * out[0] GCL tile records, out[1] GCL tiles (a row with more than 128 neighbours expands to several), out[2] GCL edges,
 * out[3] coordinate-update records.  All zero for FC graphs.  Blocking (device synchronise). For bench.py / tests. */
dl_status dl_cut_graph_stats(dl_engine* e, int64_t* out);
/* Self-test of the 3xFP16 wgmma building block (128 x 256 x 128) against an fp64 host product on random data. Blocking.
 * Returns DL_OK and writes the max abs/rel error. */
dl_status dl_selftest_tc(dl_engine* e, float* max_abs_err, float* max_rel_err);
/* Same with the B operand in the K-major (b_mn_major == 0) or the MN-major canonical layout (b_mn_major == 1; the
 * transpose-B immediate of wgmma). Any other value is DL_ERR_INVALID. */
dl_status dl_selftest_tc_layout(dl_engine* e, int32_t b_mn_major, float* max_abs_err, float* max_rel_err);

/*
 * Output stage (the step right after sample_chain in every generation script).
 *
 * dl_restore_frame -- generate.py:163-171, generate_with_pocket.py:272-280, sample.py:164-171: put the molecules back
 * to the input frame, x += (sum_n positions*com_mask / sum_n com_mask) * node_mask, in place on the first three columns
 * of `xh` (row stride `row_stride` floats: 3 for a packed x, 3+F for chain[0]).  DEVICE buffers, enqueued on `stream`.
 *   positions (B,N,3) fp32; com_mask (B,N) fp32 (fragment_mask or anchors); node_mask (B,N) int8
 */
dl_status dl_restore_frame(int32_t B, int32_t N, int32_t row_stride, float* xh, const float* positions,
                           const float* com_mask, const int8_t* node_mask, void* stream);
/* Same when the sampled batch was re-templated with sampled linker sizes (create_templates_for_linker_generation,
 * datasets.py:483-512): `xh` / `node_mask` have the template's padded length N while `positions` / `com_mask` keep the
 * input batch's padded length N_pos (generate.py:165-171 mixes exactly these two). */
dl_status dl_restore_frame2(int32_t B, int32_t N, int32_t N_pos, int32_t row_stride, float* xh, const float* positions,
                            const float* com_mask, const int8_t* node_mask, void* stream);

/*
 * dl_format_xyz -- visualizer.save_xyz_file (src/visualizer.py:14-31) for a whole batch: the text of the B .xyz files
 * ("%d\n\n" then one "%s %.9f %.9f %.9f\n" line per valid atom, symbol = symbols[argmax one_hot]) written
 * back to back into `out`; molecule b occupies out[offsets[b] .. offsets[b+1]).  HOST buffers.
 *   positions (B,N,>=3) fp32 with row stride pos_row_stride; one_hot (B,N,>=F) fp32 with row stride oh_row_stride
 *   symbols: n_symbols >= F NUL-terminated element symbols (const.IDX2ATOM / GEOM_IDX2ATOM, src/const.py:15,31)
 * Returns the number of bytes the full text needs (write again with a larger buffer if > out_cap; out may be NULL
 * for a sizing call), or a negative dl_status.
 */
int64_t dl_format_xyz(int32_t B, int32_t N, int32_t F, const float* positions, int32_t pos_row_stride,
                      const float* one_hot, int32_t oh_row_stride, const int8_t* node_mask,
                      const char* const* symbols, int32_t n_symbols, char* out, int64_t out_cap, int64_t* offsets);

/*
 * dl_bond_orders -- molecule_builder.build_xae_molecule / get_bond_order (src/molecule_builder.py:44-102) for a padded
 * batch: E[b][i][j] (i > j, both atoms valid) = 0..3 from the pair distance in pm against single / double / triple bond
 * length thresholds (table value + margin, src/const.py:66-146,180) of the type pair ordered by type index; the upper
 * triangle and masked rows are 0. The distance is torch.cdist's over the molecule's n rows with node_mask != 0, the later
 * row i first (stated at "distance" under dl_molecule_checks).  DEVICE buffers, enqueued on `stream`.
 *   x (B,N,>=3) fp32 with row stride x_row_stride; atom_types (B,N) int32; node_mask (B,N) int8
 *   thr1/thr2/thr3 (n_types,n_types) fp32 indexed [min type][max type]; negative = pair absent from that table
 *   E (B,N,N) int8 out
 */
dl_status dl_bond_orders(int32_t B, int32_t N, int32_t n_types, const float* x, int32_t x_row_stride,
                         const int32_t* atom_types, const int8_t* node_mask, const float* thr1, const float* thr2,
                         const float* thr3, int8_t* E, void* stream);

/*
 * SizeGNN (src/linker_size.py:45-91) as called by SizeClassifier.forward (src/linker_size_lightning.py:83-110): the
 * linker-size classifier that generate.py:88-99 runs once per batch before the sampler.
 *   out[b] = mean_n embedding_out( GCL_L(...GCL_1(embedding_in(one_hot*frag))) )     (B, out_node_nf) logits
 * with ReLU GCLs on the fragment atoms, edges = fragment pairs (self loops included) whose SQUARED distance is < 6
 * (linker_size_lightning.py:107-108), sum aggregation, normalization_factor 1.
 * Weight names: "embedding_in.{weight,bias}", "layer<l>.edge_mlp.{0,2}.{weight,bias}", "layer<l>.node_mlp.{0,2}.{weight,
 * bias}" (l = 0 is SizeGNN.gcl1, l >= 1 is gcl_layers[l-1]; with normalization='batch_norm' the caller folds the eval-mode
 * BatchNorm1d affine maps into node_mlp.0 / node_mlp.2), "embedding_out.{weight,bias}"; (out,in) row-major fp32, HOST.
 */
typedef struct dl_sizegnn dl_sizegnn; /* opaque */
typedef struct dl_sizegnn_config {
  int32_t in_node_nf;   /* one-hot width the network was trained with */
  int32_t hidden_nf;    /* 128 (train_size_gnn.py's default) or 256 (the README's recipe); else DL_ERR_UNSUPPORTED */
  int32_t out_node_nf;  /* number of linker-size classes */
  int32_t n_layers;     /* GCLs (train_size_gnn.py:20: 3) */
  int32_t device;
} dl_sizegnn_config;
dl_status dl_sizegnn_create(const dl_sizegnn_config* cfg, dl_sizegnn** out);
dl_status dl_sizegnn_destroy(dl_sizegnn* e);
dl_status dl_sizegnn_set_weight(dl_sizegnn* e, const char* name, const float* host_data, int64_t numel);
dl_status dl_sizegnn_finalize_weights(dl_sizegnn* e);
/* DEVICE buffers, enqueued on `stream`:
 *   xh            (B,N,3+in_node_nf) fp32: [positions | one_hot] (the kernel applies fragment_mask to both)
 *   fragment_mask (B,N) int8 0/1       (data['fragment_mask'], or 'fragment_only_mask' with pockets)
 *   edge_mask     (B,N,N) int8, non-zero = live pair (datasets.collate_with_fragment_edges, datasets.py:396-402), or NULL
 *   out           (B,out_node_nf) fp32 logits
 * N > 6144 is DL_ERR_UNSUPPORTED (the work plan's shared-memory staging; the same limit holds for every forward). */
dl_status dl_sizegnn_forward(dl_sizegnn* e, int32_t B, int32_t N, const float* xh, const int8_t* fragment_mask,
                             const int8_t* edge_mask, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DIFFLINKER_B200_H_ */
