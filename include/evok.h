/*
 * evok.h -- C ABI of libevok.so: the sm_90a kernels behind the per-generation hot path of
 * EvoTorch's distribution-based searchers (PGPE / SNES / CEM / XNES / CMA-ES).
 *
 * The reference (nnaisense/evotorch @ cebcac4f) has no FFI: its "plugin interface" on this path is a
 * set of Python methods whose bodies are sequences of torch ops.  Each entry point below replaces the
 * body of one of those methods; the citation is `path:line` under /root/reference/src/evotorch.
 * INTEGRATION.md shows the ctypes stub a maintainer of the reference would add at each site.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless its name ends in `_host`;
 *   - the caller owns all memory, including workspaces (query the *_workspace_bytes functions);
 *     the library never allocates, frees or synchronises (the one exception: evok_peer_alloc / open / close / free);
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, so every call is
 *     CUDA-graph capturable and re-entrant;
 *   - return value: 0 = ok, negative = argument error (EVOK_E_*), positive = cudaError_t;
 *   - populations are row-major fp32: X[i * ldx + j], i < n_rows, j < D.
 */
#ifndef EVOK_H_
#define EVOK_H_

#ifndef __CUDACC_RTC__ /* NVRTC compiles this header as part of evotorch_b200/csrc/evok_sampler.cuh, which defines the integer types */
#include <stddef.h>
#include <stdint.h>
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define EVOK_ABI_VERSION 1

#if defined(__GNUC__)
#define EVOK_API __attribute__((visibility("default")))
#else
#define EVOK_API
#endif

/* argument-error codes (negative return values) */
#define EVOK_E_NULLPTR (-1)
#define EVOK_E_BADSIZE (-2)
#define EVOK_E_BADENUM (-3)
#define EVOK_E_WORKSPACE (-4)
#define EVOK_E_ODDROWS (-5) /* symmetric sampling / gradients need an even number of rows */
#define EVOK_E_ALIGN (-6)
#define EVOK_E_NOKERNEL (-7) /* the cubin of a registered objective lacks one of its EVOK_OBJ_KERNELS kernels */
#define EVOK_E_NODATA (-8)   /* a registered objective that declares data was launched by its own id, not by an instance's */
#define EVOK_E_NOISEKEY (-9) /* evok_eval of an objective that draws noise: evaluate it with a key (evok_eval_keyed) */

#define EVOK_MAX_PEERS 16 /* GPUs of one NVLink domain that can take part in a peer exchange */

/* objective functions with a fused evaluation kernel */
#define EVOK_OBJ_NONE 0      /* sample only */
#define EVOK_OBJ_SPHERE 1    /* sum x^2 */
#define EVOK_OBJ_RASTRIGIN 2 /* 10 D + sum(x^2 - 10 cos(2 pi x))  (reference README.md:86-89) */
#define EVOK_OBJ_ACKLEY 3    /* -20 exp(-0.2 sqrt(mean x^2)) - exp(mean cos(2 pi x)) + 20 + e */
#define EVOK_OBJ_COUNT 4
/* objectives registered at run time (evok_objective_register) take the ids EVOK_OBJ_USER_BASE, EVOK_OBJ_USER_BASE + 1, ...
 * in registration order, at most EVOK_OBJ_USER_CAPACITY of them per process; every id in between is EVOK_E_BADENUM */
#define EVOK_OBJ_USER_BASE 64
#define EVOK_OBJ_USER_CAPACITY 256
/* instances of registered objectives that declare data (evok_objective_instance) take ids from EVOK_OBJ_INSTANCE_BASE; a
 * released id is reused, and at most EVOK_OBJ_INSTANCE_CAPACITY are alive at a time */
#define EVOK_OBJ_INSTANCE_BASE 1024
#define EVOK_OBJ_INSTANCE_CAPACITY 65536
#define EVOK_MAX_DATA 4 /* data names (float32 vectors of the row length and scalars) of one objective */

/* ranking methods (tools/ranking.py:186) */
#define EVOK_RANK_CENTERED 0
#define EVOK_RANK_LINEAR 1
#define EVOK_RANK_NES 2
#define EVOK_RANK_NORMALIZED 3
#define EVOK_RANK_RAW 4

/* gradient forms: S1_j = sum_r a_r eps_rj ; S2_j = sum_r b_r g(eps_rj) */
#define EVOK_GRAD_SEPARABLE 0 /* g = (eps^2 - sigma^2)/sigma; a=b=w_i; all rows      (distributions.py:548-579) */
#define EVOK_GRAD_SYMMETRIC 1 /* same g; a,b = (w+ -/+ w-)/2; even rows only           (distributions.py:708-773) */
#define EVOK_GRAD_EXP 2       /* g = (eps/sigma)^2 - 1; a=b=w_i                        (distributions.py:783-793) */
#define EVOK_GRAD_MOMENTS 3   /* g = eps^2; a=b=w_i (0/1 elite mask for CEM)           (distributions.py:538-546) */

int evok_abi_version(void);
/* number of kernels launched by this library since it was loaded (for bench.py's gpu_launches) */
uint64_t evok_launch_count(void);
const char* evok_error_string(int code);

/* ---------------------------------------------------------------------------------------------
 * K1 / K2: population sampling and evaluation.
 * Replaces: Distribution.sample -> SymmetricSeparableGaussian._fill / SeparableGaussian._fill
 *           (distributions.py:155-216, :514, :705) -> make_gaussian (tools/misc.py:1663-1755), and, for the
 *           built-in objectives, Problem._evaluate_batch (core.py:2602-2608).
 * Random numbers: Philox4x32-10 keyed by `seed`; the counter of a draw is a pure function of
 * (global row or direction index, column, `stream_id`), so the population does not depend on the launch
 * geometry nor on how rows are sharded over GPUs (`row0` = global index of the first local row).
 * symmetric != 0: rows 2k and 2k+1 are mu + sigma*z_k and mu - sigma*z_k (row0 and n_rows even).
 * X may be NULL when objective != NONE ("lazy population": evaluate without materialising).
 * f may be NULL when objective == NONE.
 * stream_offset_dev (nullable): device pointer to a 32-bit generation counter that is ADDED to the low word of
 * stream_id when the kernel runs -- a CUDA graph captured once then draws a fresh population at every replay
 * (the host increments the counter with an in-graph kernel); NULL = use stream_id as is.
 */
int evok_sample_eval(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0,
                     int64_t n_rows, int64_t D, int symmetric, uint64_t seed, uint64_t stream_id,
                     const uint32_t* stream_offset_dev, float* f, void* stream);

/* K2 alone: f[i] = objective(X[i, :]) for an already materialised population (torch-RNG parity mode,
 * CMA-ES / XNES populations).  Replaces the user's vectorised torch objective at core.py:2604. */
int evok_eval(int objective, const float* X, int64_t ldx, int64_t n_rows, int64_t D, float* f, void* stream);

/* K2 with the Philox draw of the rows: row i of X is global row (row0 + i) of the draw (seed, stream_id, stream_offset_dev as in
 * evok_sample_eval).  An objective whose expressions draw noise (evok_objective_declare_noise) takes its rand() / randn() from
 * that draw, so a row that evok_sample_eval sampled with the same arguments gets the same fitness bit for bit on the vectorised
 * path; evok_eval refuses such an objective (EVOK_E_NOISEKEY) and launches nothing, rather than evaluate it with a fixed key.
 * For an objective without noise it is evok_eval: the same kernel and the same bits.  Errors: those of evok_eval, and
 * EVOK_E_BADSIZE for row0 < 0. */
int evok_eval_keyed(int objective, const float* X, int64_t ldx, int64_t row0, int64_t n_rows, int64_t D, uint64_t seed, uint64_t stream_id,
                    const uint32_t* stream_offset_dev, float* f, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Objectives defined at run time (evotorch_b200/jit.py compiles them with NVRTC from csrc/evok_sampler.cuh).
 * evok_objective_register takes an sm_90a cubin and the lowered names of its EVOK_OBJ_KERNELS kernels, in this order:
 *   EVOK_OBJ_KERNEL_SAMPLE + 4 sym + 2 store + vec : sample_eval_kernel<Acc, sym, store, vec, PUSH = false, SQ = false>
 *   EVOK_OBJ_KERNEL_PUSH   + 4 sym + 2 store + vec : sample_eval_kernel<Acc, sym, store, vec, PUSH = true,  SQ = false>
 *   EVOK_OBJ_KERNEL_SQ     + 2 store + vec         : sample_eval_kernel<Acc, false, store, vec, PUSH = false, SQ = true>
 *   EVOK_OBJ_KERNEL_EVAL   + vec                   : eval_kernel<Acc, vec>
 * The fitness of a row is Acc's function of sums over the row's elements x_j and, for an Acc with pair terms (kPairs), over
 * its neighbour pairs (x_j, x_{j+1}), j = 0 .. D-2; the kernels fold each element and each pair exactly once.
 * It copies the image and the names, writes the new id to *id_out_host and needs no device.  The id is then accepted by
 * evok_sample_eval, evok_sample_eval_sq, evok_sample_eval_push and evok_eval, which launch the registered kernels exactly
 * as they launch a built-in objective's (same argument checks, kernel choice and grid).
 * The module is loaded on a device by the first call that uses the id there, or by evok_objective_load (on the current
 * device), which a caller about to capture a CUDA graph uses to keep the loading out of the capture.  A cubin without one
 * of the kernels yields EVOK_E_NOKERNEL from every call on that device, and nothing is launched.
 * Errors: EVOK_E_NULLPTR, EVOK_E_BADSIZE (bytes == 0, n_kernels != EVOK_OBJ_KERNELS, registry full), EVOK_E_BADENUM
 * (evok_objective_load of an id that is neither registered nor a live instance; an instance id loads its base).
 * --------------------------------------------------------------------------------------------- */
#define EVOK_OBJ_KERNEL_SAMPLE 0
#define EVOK_OBJ_KERNEL_PUSH 8
#define EVOK_OBJ_KERNEL_SQ 16
#define EVOK_OBJ_KERNEL_EVAL 20
#define EVOK_OBJ_KERNELS 22
int evok_objective_register(const void* cubin, size_t bytes, const char* const* kernel_names_host, int n_kernels, int* id_out_host);
int evok_objective_load(int objective);

/* The batched sampler of an objective (evok_sample_eval_batched) is a second family of kernels, kept in a second image so
 * that a registered objective that never runs batched searches compiles and loads only the EVOK_OBJ_KERNELS above:
 *   EVOK_OBJ_KERNEL_BATCHED + 4 sym + 2 store + vec : sample_eval_batched_kernel<Acc, sym, store, vec>
 * evok_objective_register_batched attaches the sm_90a cubin of these EVOK_OBJ_BATCHED_KERNELS kernels (lowered names in this
 * order, positions counted from EVOK_OBJ_KERNEL_BATCHED) to the registered id `objective`.  It copies the image and the names
 * and needs no device; the module is loaded on a device by the first batched call there.  Attaching again replaces the image
 * for the devices that have not loaded it yet.  A registered id without a batched image yields EVOK_E_NOKERNEL from
 * evok_sample_eval_batched, which then launches nothing.
 * Errors: EVOK_E_NULLPTR, EVOK_E_BADSIZE (bytes == 0, n_kernels != EVOK_OBJ_BATCHED_KERNELS), EVOK_E_BADENUM (`objective` is
 * a built-in id or is not registered). */
#define EVOK_OBJ_KERNEL_BATCHED 22
#define EVOK_OBJ_BATCHED_KERNELS 8
int evok_objective_register_batched(int objective, const void* cubin, size_t bytes, const char* const* kernel_names_host, int n_kernels);

/* The batched evaluation of an objective (evok_eval_batched) is a third family, in a third image, so that a registered objective
 * that never evaluates batched populations compiles and loads neither it nor the batched samplers:
 *   EVOK_OBJ_KERNEL_EVAL_BATCHED + vec : eval_batched_kernel<Acc, vec>
 * evok_objective_register_eval_batched attaches the sm_90a cubin of these EVOK_OBJ_EVAL_BATCHED_KERNELS kernels (lowered names in
 * this order, positions counted from EVOK_OBJ_KERNEL_EVAL_BATCHED) to the registered id `objective`, as
 * evok_objective_register_batched does for the batched samplers; the module is loaded on a device by the first
 * evok_eval_batched there.  A registered id without this image yields EVOK_E_NOKERNEL from evok_eval_batched.
 * Errors: EVOK_E_NULLPTR, EVOK_E_BADSIZE (bytes == 0, n_kernels != EVOK_OBJ_EVAL_BATCHED_KERNELS), EVOK_E_BADENUM (`objective`
 * is a built-in id or is not registered). */
#define EVOK_OBJ_KERNEL_EVAL_BATCHED 30
#define EVOK_OBJ_EVAL_BATCHED_KERNELS 2
int evok_objective_register_eval_batched(int objective, const void* cubin, size_t bytes, const char* const* kernel_names_host, int n_kernels);

/* Transformed objectives: an accumulator with kTransform (csrc/evok_sampler.cuh) whose terms read y = M (x - o) of each row as well
 * as x.  Its sampler kernels cannot exist (a sampler produces a row one column group at a time, y needs the whole row), so it is
 * registered with a fourth family only, evaluated by evok_eval_transform_batched:
 *   EVOK_OBJ_KERNEL_TRANSFORM     + vec : eval_transform_fused_kernel<Acc, vec>  (small D: y on the CUDA cores in shared memory)
 *   EVOK_OBJ_KERNEL_TRANSFORM + 2 + vec : eval_transform_kernel<Acc, vec>        (large D: y from the batched 3xTF32 GEMM)
 * evok_objective_register_transform takes the sm_90a cubin of these EVOK_OBJ_TRANSFORM_KERNELS kernels (lowered names in this order)
 * and writes a new id to *id_out_host, as evok_objective_register does; it needs no device.  evok_objective_declare_data and
 * _declare_noise and evok_objective_instance apply to it as to any registered id; every other entry point that takes an objective
 * yields EVOK_E_NOKERNEL for it, and evok_eval_transform_batched yields EVOK_E_NOKERNEL for every id without this family.
 * Errors: EVOK_E_NULLPTR, EVOK_E_BADSIZE (bytes == 0, n_kernels != EVOK_OBJ_TRANSFORM_KERNELS, registry full). */
#define EVOK_OBJ_KERNEL_TRANSFORM 32
#define EVOK_OBJ_TRANSFORM_KERNELS 4
int evok_objective_register_transform(const void* cubin, size_t bytes, const char* const* kernel_names_host, int n_kernels, int* id_out_host);

/* Objectives with noise.  The accumulator of a registered objective may draw uniform and normal noise from the Philox key of
 * the population it evaluates (kNoise in csrc/evok_sampler.cuh); its eval_kernel<Acc, vec> then takes the draw of the rows as
 * its last argument.  evok_objective_declare_noise tells the library so, right after
 * evok_objective_register: from then on evok_eval refuses the id (and its instances) with EVOK_E_NOISEKEY and evok_eval_keyed
 * passes the key.  The samplers need nothing more: they draw the noise from the key they sample with.
 * Errors: EVOK_E_BADENUM (`objective` is not a registered id). */
int evok_objective_declare_noise(int objective);

/* Objectives with data.  The accumulator of a registered objective may read up to EVOK_MAX_DATA float32 device arrays (kData in
 * csrc/evok_sampler.cuh): vectors with one entry per column of a row, and scalars.  Which name is which is part of its source;
 * the arrays are not.  evok_objective_declare_data tells the library so, right after evok_objective_register and before the id
 * is used: is_vector_host[i] != 0 makes data name i a vector.  From then on the id itself launches nothing (EVOK_E_NODATA):
 * evok_objective_instance makes an id that shares the kernel images and per-device kernel tables of `base` and carries its own
 * binding, and every entry point that takes an objective id takes it, with its signature unchanged.  The binding reaches the
 * kernel as a launch argument (captured by value in a CUDA graph), so instances of one base never interfere, on any streams.
 *   ptrs_host[i]         device array of data name i of the first item; the library keeps the pointer, the caller keeps the
 *                        array alive and in place until evok_objective_release.  Writing new values into it on a stream takes
 *                        effect on the launches (and graph replays) that follow on that stream.
 *   lens_host[i]         1 for a scalar; for a vector its length, which must equal D of every call (EVOK_E_BADSIZE there)
 *   n_items              1: every call, batched or not, uses the one binding.  > 1: item b of evok_sample_eval_batched reads
 *                        ptrs_host[i] + b * item_strides_host[i] (a stride may be 0: that name is shared); n_items must then be
 *                        the n_items of the call, and every non-batched entry refuses the id (EVOK_E_BADSIZE).
 * The vectorised kernels read a vector with 16-byte loads: they are chosen only if every vector's ptrs_host[i] is 16-byte
 * aligned and, with n_items > 1, its item stride is a multiple of 4; else the call runs the scalar-column kernels.
 * The data checks of a launch come after the entry point's own, and nothing is launched when one fails.
 * evok_objective_release frees an instance id (kernels already enqueued keep their copy of the binding).
 * Errors: EVOK_E_NULLPTR; EVOK_E_BADENUM (`objective` / `base` is not a registered id, `id` is not a live instance);
 * EVOK_E_BADSIZE (n_data outside 1 .. EVOK_MAX_DATA or, for an instance, not the declared count; data declared twice; a length
 * < 1, or 1 for a declared vector, or > 1 for a declared scalar; n_items < 1; a negative stride; EVOK_OBJ_INSTANCE_CAPACITY
 * instances alive); EVOK_E_NODATA (`base` declares no data). */
int evok_objective_declare_data(int objective, int n_data, const int* is_vector_host);
int evok_objective_instance(int base, const float* const* ptrs_host, const int64_t* lens_host, const int64_t* item_strides_host,
                            int64_t n_items, int n_data, int* id_out_host);
int evok_objective_release(int id);

/* ---------------------------------------------------------------------------------------------
 * K3: fitness -> utilities.  Replaces tools/ranking.py:24-183 (`rank` :189).
 * Sort semantics: STABLE (equal fitnesses keep ascending index order), -0 == +0, NaN largest;
 * identical to torch.argsort(f, descending=!higher_is_better, stable=True).
 * w: utilities (same length).  perm (nullable): the sorted order, worst first, as int64 (what
 * `argsort` returns).  ws: workspace of at least evok_rank_workspace_bytes(N) bytes.
 * Implementation: N <= 8192 -> ONE launch (rank by counting, utilities / flags / permutation written by the same kernel);
 * larger N -> stable LSD radix sort (4 passes x 8 bits) + a scatter kernel.  Both produce bit-identical results.
 * --------------------------------------------------------------------------------------------- */
size_t evok_rank_workspace_bytes(int64_t N);
int evok_rank(int method, const float* f, int64_t N, int higher_is_better, float* w, int64_t* perm, void* ws,
              size_t ws_bytes, void* stream);

/* Stable argsort of fp32 keys (SolutionBatch.argsort core.py:3827, CEM elite selection distributions.py:541,
 * CMA-ES cmaes.py:445).  Same workspace as evok_rank. */
int evok_argsort(const float* keys, int64_t N, int descending, int64_t* perm, void* ws, size_t ws_bytes,
                 void* stream);

/* out[i] = table[position of keys[i] in the stable sorted order] -- "the weight of a solution is weights[its rank]"
 * (CMA-ES get_population_weights, cmaes.py:445-451: argsort, inverse-permutation scatter and gather, in one call).
 * descending != 0: position 0 is the largest key.  Same workspace as evok_rank. */
int evok_rank_table(const float* keys, int64_t N, int descending, const float* table, float* out, void* ws, size_t ws_bytes, void* stream);

/* In-place weight post-processing on the N-vector (distributions.py:562-563, :722-723 `w - mean(w)`;
 * :784-785 `w / sum|w|`).  mode 1: subtract mean; mode 2: divide by sum of absolute values. */
int evok_weights_adjust(float* w, int64_t N, int mode, void* stream);

/* 0/1 mask of the `num_elites` largest weights, ties broken by ascending index (distributions.py:540-542).
 * Needs the rank workspace. */
int evok_elite_mask(const float* w, int64_t N, int64_t num_elites, float* mask, void* ws, size_t ws_bytes,
                    void* stream);

/* ---------------------------------------------------------------------------------------------
 * K4: utility-weighted column reductions over the population.
 * Replaces SeparableGaussian._compute_gradients (distributions.py:548-579),
 * SymmetricSeparableGaussian._compute_gradients (:708-773), ExpSeparableGaussian._compute_gradients
 * (:783-793) and the elite moments of _compute_gradients_via_parenthood_ratio (:538-546).
 *   out_mu[j]    = scale_mu    * sum_r a_r * (X[r,j] - mu[j])
 *   out_sigma[j] = scale_sigma * sum_r b_r * g(X[r,j] - mu[j])          (g, a, b per `form` above)
 * `w` holds the weights of the n_rows local rows (a slice of the global utility vector when the
 * population is sharded; the partial results of the shards then add up: all-reduce(sum)).
 * Deterministic (fixed two-stage reduction order, no atomics).
 * --------------------------------------------------------------------------------------------- */
size_t evok_grad_workspace_bytes(int64_t n_rows, int64_t D);
int evok_grad(int form, const float* X, int64_t ldx, const float* w, const float* mu, const float* sigma,
              int64_t n_rows, int64_t D, float scale_mu, float scale_sigma, float* out_mu, float* out_sigma,
              void* ws, size_t ws_bytes, void* stream);

/* K4 without a materialised population: regenerates eps from the Philox counters used by
 * evok_sample_eval(..., X = NULL) with the same (seed, stream_id, row0). */
int evok_grad_regen(int form, const float* w, const float* mu, const float* sigma, int64_t row0, int64_t n_rows,
                    int64_t D, uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev, float scale_mu,
                    float scale_sigma, float* out_mu, float* out_sigma, void* ws, size_t ws_bytes, void* stream);

/* evok_grad over a materialised population X that evok_sample_eval wrote from this mu and sigma with the same (seed,
 * stream_id, stream_offset_dev, row0): part of the rows are rebuilt from their Philox counters on the SMs while the rest
 * stream from X, which cuts the bytes read.  The result is bit-identical to evok_grad for every split.
 * split = rebuilt row groups per 16 (0 = read every row, 16 = rebuild every row, -1 = the library's choice).  Shapes the
 * TMA-staged kernel does not take (D % 4, alignment, D < 512, fewer than 4096 units, EVOK_GRAD_MOMENTS) read every row. */
int evok_grad_hybrid(int form, const float* X, int64_t ldx, const float* w, const float* mu, const float* sigma, int64_t row0,
                     int64_t n_rows, int64_t D, uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev, int split,
                     float scale_mu, float scale_sigma, float* out_mu, float* out_sigma, void* ws, size_t ws_bytes, void* stream);

/* The split evok_grad_hybrid uses for split = -1 on a card whose enforced power limit is power_limit_mw milliwatts
 * (<= 0: unknown, which takes the value of a power-capped card).  The choice is made once per device. */
int evok_grad_auto_split(int64_t power_limit_mw);

/* The enforced power limit of CUDA device `device` in milliwatts, read through NVML, or -1 when it cannot be read. */
int64_t evok_grad_power_limit_mw(int device);

/* ---------------------------------------------------------------------------------------------
 * K5: D-vector updates (no host synchronisation; norms are reduced on the device).
 * --------------------------------------------------------------------------------------------- */
/* ClipUp.ascent (optimizers.py:319-357): v <- clip(momentum*v + stepsize*g/||g||, max_speed).
 * velocity is updated in place; step_out (nullable) receives the ascent step; mu (nullable) += step. */
int evok_clipup_step(const float* g, int64_t D, float* velocity, float stepsize, float momentum, float max_speed,
                     float* step_out, float* mu, void* stream);
/* Adam via TorchOptimizer.ascent (optimizers.py:60-91, :101-165): m, v updated in place; `t` is the 1-based
 * step count; step = lr * m_hat / (sqrt(v_hat) + eps). */
int evok_adam_step(const float* g, int64_t D, float* m, float* v, int64_t t, float lr, float beta1, float beta2,
                   float eps, float* step_out, float* mu, void* stream);
/* SGD with optional momentum (optimizers.py:168-228): buf <- momentum*buf + g (first step: buf = g). */
int evok_sgd_step(const float* g, int64_t D, float* buf, int first_step, float lr, float momentum, float* step_out,
                  float* mu, void* stream);
/* mu += lr * g  (Distribution._follow_gradient with a plain learning rate, distributions.py:385). */
int evok_axpy(const float* g, int64_t D, float lr, float* mu, void* stream);

/* sigma update + controlled clamp.  Replaces distributions.py:591-596 / :805-808 and modify_tensor
 * (tools/misc.py:711-816) as used by gaussian.py:404-416.
 *   exp_form == 0: target = sigma + lr*g          exp_form != 0: target = sigma * exp(0.5*lr*g)
 *   lo = max(lb, sigma - |sigma|*mc), hi = min(ub, sigma + |sigma|*mc); sigma <- min(max(target, lo), hi)
 * lb / ub / mc: device vectors (length D) or NULL; when NULL the scalar is used; a NaN scalar means
 * "not set" (-inf / +inf / no max-change limit).  max / min are torch.max / torch.min: a NaN in any operand that is
 * set (target, a vector entry, |sigma|*mc = 0*inf) makes the result NaN. */
int evok_sigma_update(float* sigma, const float* g, int64_t D, float lr, int exp_form, const float* lb_vec,
                      float lb, const float* ub_vec, float ub, const float* mc_vec, float mc, void* stream);

/* CEM finalisation from elite moments (distributions.py:543-546): given S1 = sum eps, S2 = sum eps^2 over
 * the E elites, writes grad_mu = S1/E and grad_sigma = sqrt(max((S2 - S1^2/E)/(E-1), 0)) - sigma.  As torch.std of
 * E < 2 rows, E = 1 gives grad_sigma = NaN and E = 0 NaN in both; a NaN variance stays NaN (torch.clamp_min). */
int evok_cem_finalize(const float* s1, const float* s2, const float* sigma, int64_t D, int64_t num_elites,
                      float* grad_mu, float* grad_sigma, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K8: batched flat-parameter MLP policy forward, one observation per policy.
 * Replaces Policy.__call__ (neuroevolution/net/vecrl.py:1240-1279: vmap(functional_call) over the rows of the
 * N x L parameter matrix set by set_parameters) for feed-forward nets made of Linear layers + activations.
 * Parameter row layout (net/functional.py:118-129): per layer W (out x in, row-major) then b (out).
 *   out[i, :] = layer_{n-1}(... act_0(W_0 obs[i, :] + b_0) ...)        acts: EVOK_ACT_* applied after each layer
 * dims_host: n_layers + 1 layer widths (host array); acts_host: n_layers activation ids (host array).
 * --------------------------------------------------------------------------------------------- */
#define EVOK_ACT_NONE 0
#define EVOK_ACT_TANH 1
#define EVOK_ACT_RELU 2
#define EVOK_ACT_SIGMOID 3
int64_t evok_mlp_parameter_length(int n_layers, const int32_t* dims_host);
int evok_mlp_forward(const float* params, int64_t ldp, const float* obs, int64_t ldo, float* out, int64_t ldout, int64_t N,
                     int n_layers, const int32_t* dims_host, const int32_t* acts_host, void* stream);

/* The same forward with the observation pre-processing of the rollout loop fused into the observation load
 * (vecgymne.py:604-660, :822-836; net/runningnorm.py:412-533): x = clamp((obs - mean) / stdev, clip_lo, clip_hi), where
 * mean = obs_sum / count and stdev = sqrt(max(obs_sumsq / count - mean^2, min_variance)) come from the RunningNorm sums on the
 * device (obs_sum == NULL: no normalisation; clip_* = NaN: no clipping).  `active` (N bytes, nullable): policies whose flag
 * is 0 are skipped -- their parameters are never read -- and receive zero actions.  `ws` (nullable, >= 4 bytes, 4-byte aligned):
 * with a mask, CTAs draw row chunks from a work counter kept there instead of a static round-robin (which leaves the number of
 * surviving policies per CTA binomially unbalanced). */
int evok_mlp_forward_prep(const float* params, int64_t ldp, const float* obs, int64_t ldo, float* out, int64_t ldout, int64_t N,
                          int n_layers, const int32_t* dims_host, const int32_t* acts_host, const float* obs_sum, const float* obs_sumsq,
                          const int64_t* obs_count_dev, float min_variance, float clip_lo, float clip_hi, const uint8_t* active,
                          void* ws, size_t ws_bytes, void* stream);

/* The forward of N networks on ONE shared input batch (B x dims[0]) -- a population scored on a common minibatch
 * (neuroevolution/supervisedne.py:337-347, where the reference loops over the solutions: parameterize_net + network(x), neproblem.py:342,
 * supervisedne.py:250).  Here the first layer of ALL networks is one tensor-core product of the stacked weight rows with the shared batch
 * (evok_gemm_gather_rows: the weight rows are gathered from the flat parameter rows -- any 4-byte alignment -- straight into the swizzled
 * operand tiles, so every parameter is read from HBM once; bias and activation in the epilogue), the remaining (small, per-network)
 * layers run in a second kernel on the staged activations.  out: [N][B][dims[n_layers]].  n_layers >= 2, hidden widths <= 512,
 * X 16-byte aligned with ldx % 4 == 0.  evok_mlp_forward_shared_supported: 1 if evok_mlp_forward_shared takes these layer widths,
 * 0 if it would return EVOK_E_BADSIZE (also when a layer after the first is too wide for its second kernel to stage in shared memory:
 * e.g. 8-256-256-2 or 8-512-34); needs no device. */
int evok_mlp_forward_shared_supported(int n_layers, const int32_t* dims_host);
size_t evok_mlp_forward_shared_workspace_bytes(int64_t N, int64_t B, int n_layers, const int32_t* dims_host);
int evok_mlp_forward_shared(const float* params, int64_t ldp, int64_t N, const float* X, int64_t ldx, int64_t B, int n_layers,
                            const int32_t* dims_host, const int32_t* acts_host, float* out, void* ws, size_t ws_bytes, void* stream);
/* C[(i, h), b] = act(sum_k W_i[h, k] X[b, k] + bias_i[h]),  W_i = params + i * batch_stride + w_offset (rows_per_batch x K, row-major),
 * bias_i = params + i * batch_stride + bias_offset (bias_offset < 0: none).  3xTF32 on wgmma, fp32 accuracy. */
int evok_gemm_gather_rows(const float* params, int64_t batch_stride, int64_t w_offset, int64_t rows_per_batch, int64_t n_batches, const float* X,
                          int64_t ldx, int64_t n_cols, int64_t K, int64_t bias_offset, int act, float* C, int64_t ldc, void* stream);
/* The same product on the PERSISTENT kernel (one CTA per SM walks the tiles; X pre-split into hi / lo copies in `ws`, so X may have any
 * alignment; epilogue overlapped with the next tile).  unit_fastest != 0: C[(batch * n_cols + col) * rows_per_batch + row] (ldc unused)
 * instead of C[(batch * rows_per_batch + row) * ldc + col].  Used by evok_mlp_forward_shared. */
size_t evok_gemm_gather_rows_workspace_bytes(int64_t n_cols, int64_t K);
int evok_gemm_gather_rows_ws(const float* params, int64_t batch_stride, int64_t w_offset, int64_t rows_per_batch, int64_t n_batches, const float* X,
                             int64_t ldx, int64_t n_cols, int64_t K, int64_t bias_offset, int act, float* C, int64_t ldc, int unit_fastest, void* ws,
                             size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K6 / K7: fp32-accurate tensor-core GEMM (wgmma + TMA, 3xTF32 operand splitting).
 *   C[M x N] = A[M x K] * B[N x K]^T        A, B, C row-major fp32 (lda, ldb >= K; ldc >= N)
 *   optional C2[M x N] = alpha_dev[0] * (A B^T) + bias[col]    (C2 / alpha_dev / bias nullable)
 * Replaces the dense contractions of CMA-ES: `ys = (A @ zs.T).T`, `xs = m + sigma * ys` (cmaes.py:427-429; call with
 * A = zs, B = A_chol, C = ys, C2 = xs, alpha_dev = &sigma, bias = m) and the rank-mu update
 * sum_i w_i y_i y_i^T (cmaes.py:548; call with A = (w * Y)^T, B = Y^T built by evok_transpose_scale), and XNES'
 * `A z^T` / sum_i w_i z_i z_i^T (distributions.py:938, :980-984).
 * --------------------------------------------------------------------------------------------- */
size_t evok_gemm_workspace_bytes(int64_t M, int64_t N, int64_t K);
int evok_gemm_nt(const float* A, int64_t lda, const float* B, int64_t ldb, int64_t M, int64_t N, int64_t K, float* C, int64_t ldc,
                 float* C2, int64_t ldc2, const float* alpha_dev, const float* bias, void* ws, size_t ws_bytes, void* stream);
/* The same product with a fused affine update of the output (no second pass over C):
 *   C[i][j] = k[0] * (A B^T)[i][j] + k[1] * E[i][j] + k[2] * u[i] * u[j]        k_dev: 3 device floats; E, u nullable (u needs M == N)
 * E may be C itself.  Replaces the covariance update of CMA-ES, cmaes.py:519-553:
 *   C <- C + c1a (pc pc^T - C) + c_mu (Y^T diag(w) Y - sum(w) C)   with k = (c_mu, 1 - c1a - c_mu sum(w), c1a * weighted_pc^2), u = p_c. */
int evok_gemm_nt_affine(const float* A, int64_t lda, const float* B, int64_t ldb, int64_t M, int64_t N, int64_t K, float* C, int64_t ldc,
                        const float* k_dev, const float* E, int64_t lde, const float* u, void* ws, size_t ws_bytes, void* stream);
/* out[c, r] = (w ? w[r] : 1) * in[r, c]: builds the K-major operands of the weighted SYRK */
int evok_transpose_scale(const float* in, int64_t ldi, int64_t rows, int64_t cols, const float* w, float* out, int64_t ldo, void* stream);
/* both SYRK operands in one pass over `in`:  out_w[c, r] = w[r] * in[r, c],  out_p[c, r] = in[r, c] */
int evok_transpose_pair(const float* in, int64_t ldi, int64_t rows, int64_t cols, const float* w, float* out_w, float* out_p, int64_t ldo,
                        void* stream);

/* Batched K6 / K7: n_items independent products C_b = A_b B_b^T (M x N x K each) in one launch per 65535 items (grid z = item).
 * Operand b of A is at A + b * item_stride_a (item_stride_a = 0: one A shared by every item), likewise B; C_b at C + b * item_stride_c
 * (outputs are per item: item_stride_c >= (M - 1) ldc + N when n_items > 1).  A batched product never splits K, so every item is
 * summed in the order of evok_gemm_nt with a one-split plan and gets its bits.  Operands with a 16-byte aligned base, row pitch and
 * item pitch (and items that do not overlap) are read once by the GEMM through rank-3 tensor maps [items][rows][K] (rows past M / N
 * read as zeros per item); otherwise both are first split into hi / lo copies in `ws`
 * (evok_gemm_nt_batched_workspace_bytes, which takes the same operands).
 *   evok_gemm_nt_batched        : optional C2_b = alpha_b * C_b + bias_b[col] with alpha at alpha_dev + b * item_stride_alpha and bias at
 *                                 bias + b * item_stride_bias (0 = shared).  CMA-ES sampling x = m_b + sigma_b z A_b^T.
 *   evok_gemm_nt_affine_batched : C_b = k_b[0] A_b B_b^T + k_b[1] E_b + k_b[2] u_b u_b^T with k_b, E_b, u_b at their item strides (E may
 *                                 be C).  The CMA-ES covariance update of a batch of searches.
 *   evok_transpose_pair_batched : evok_transpose_pair per item (in, w, out_w / out_p at their item strides; one launch per 65535 items). */
size_t evok_gemm_nt_batched_workspace_bytes(const float* A, int64_t lda, int64_t item_stride_a, const float* B, int64_t ldb, int64_t item_stride_b,
                                            int64_t n_items, int64_t M, int64_t N, int64_t K);
int evok_gemm_nt_batched(const float* A, int64_t lda, int64_t item_stride_a, const float* B, int64_t ldb, int64_t item_stride_b, int64_t n_items,
                         int64_t M, int64_t N, int64_t K, float* C, int64_t ldc, int64_t item_stride_c, float* C2, int64_t ldc2, int64_t item_stride_c2,
                         const float* alpha_dev, int64_t item_stride_alpha, const float* bias, int64_t item_stride_bias, void* ws, size_t ws_bytes,
                         void* stream);
int evok_gemm_nt_affine_batched(const float* A, int64_t lda, int64_t item_stride_a, const float* B, int64_t ldb, int64_t item_stride_b,
                                int64_t n_items, int64_t M, int64_t N, int64_t K, float* C, int64_t ldc, int64_t item_stride_c, const float* k_dev,
                                int64_t item_stride_k, const float* E, int64_t lde, int64_t item_stride_e, const float* u, int64_t item_stride_u,
                                void* ws, size_t ws_bytes, void* stream);
int evok_transpose_pair_batched(const float* in, int64_t ldi, int64_t item_stride_in, int64_t rows, int64_t cols, const float* w,
                                int64_t item_stride_w, float* out_w, float* out_p, int64_t ldo, int64_t item_stride_out, int64_t n_items,
                                void* stream);

/* ---------------------------------------------------------------------------------------------
 * Batched searches: the functional ask / tell API with leading batch dimensions (algorithms/functional/funcpgpe.py:67, :301, :330,
 * funccem.py, funcclipup.py:95-108; `expects_ndim`, decorators.py:613).  n_items independent searches of the same shape run in ONE
 * launch per stage (grid y / z = item) instead of one launch chain per item; above 65535 items (the grid y / z limit) a stage runs
 * as item chunks of at most 65535, in order on the stream, reusing one workspace.  Tensors are contiguous [items][...] unless an item
 * stride is given (stride 0 = the operand is shared by all items).  Per-item scalar hyper-parameters are HOST arrays (they travel in
 * the launch parameters).  Every stage computes exactly what its single-search entry point computes per item.
 * --------------------------------------------------------------------------------------------- */
/* K1: item b draws with Philox stream (stream_id0 + b): same bits as evok_sample_eval(..., stream_id = stream_id0 + b) per item.
 * Launches the EVOK_OBJ_NONE kernels of the batched family (grid y = item, grid x = the resident CTAs of the kernel shared over
 * the items of a launch, at least 1 and at most what the rows need). */
int evok_sample_batched(float* X, int64_t item_stride_x, int64_t ldx, const float* mu, int64_t item_stride_mu, const float* sigma,
                        int64_t item_stride_sigma, int64_t n_items, int64_t n_rows, int64_t D, int symmetric, uint64_t seed, uint64_t stream_id0,
                        void* stream);
/* K1+K2 for a batch of searches in one launch per 65535 items: item b samples with Philox stream (stream_id0 + b) and writes its
 * n_rows fitnesses to f[b * n_rows ...] (f: [items][n_rows], contiguous).  For every item, X and f are bit-identical to
 * evok_sample_eval(objective, ..., row0 = 0, stream_id = stream_id0 + b) on that item's operands, and X to evok_sample_batched.
 * objective: a built-in id other than EVOK_OBJ_NONE (which goes through evok_sample_batched), or a registered id with a batched
 * image (evok_objective_register_batched; else EVOK_E_NOKERNEL).  X may be NULL: a lazy population, evaluated and not stored
 * (evok_grad_batched_regen rebuilds the rows its gradient needs).  Errors in this order: EVOK_E_NULLPTR (mu, sigma, f),
 * EVOK_E_BADENUM, EVOK_E_BADSIZE (negative counts or strides, D <= 0, ldx < D with X), EVOK_E_ODDROWS, EVOK_E_NOKERNEL. */
int evok_sample_eval_batched(int objective, float* X, int64_t item_stride_x, int64_t ldx, const float* mu, int64_t item_stride_mu,
                             const float* sigma, int64_t item_stride_sigma, int64_t n_items, int64_t n_rows, int64_t D, int symmetric,
                             uint64_t seed, uint64_t stream_id0, float* f, void* stream);
/* K2 for a batch of populations in one launch per 65535 items (the populations of a full-covariance CMA-ES, or values a caller
 * asked, repaired or injected): item b evaluates the n_rows rows of X + b * item_stride_x (row pitch ldx; item_stride_x = 0: every
 * item evaluates the same rows) with item b of the objective's data and writes f[b * n_rows ...] (f: [items][n_rows],
 * contiguous).  Per item, f is bit-identical to evok_eval_keyed(objective, X + b * item_stride_x, ldx, row0 = 0, n_rows, D, seed,
 * stream_id0 + b, NULL, ...) on the same path (the vectorised one needs D % 4 == 0, a 16-byte aligned X, ldx and item_stride_x
 * multiples of 4 and the data vectors' alignment of evok_objective_instance).  Only an objective with noise uses the key: row r of
 * item b then gets the noise that evok_sample_eval_batched(..., seed, stream_id0) gives row r of item b, so a population it stored
 * gets its fitnesses again.  An instance with per-item data (n_items > 1) gives item b its item b.
 * objective: a built-in id other than EVOK_OBJ_NONE, or a registered id with its batched evaluation image
 * (evok_objective_register_eval_batched), or an instance of one.  Grid: y = item, x = the resident CTAs of the kernel shared over
 * the items of a launch, at least 1 and at most what the rows need; zero items or zero rows launch nothing.
 * Errors in this order: EVOK_E_NULLPTR (X, f), EVOK_E_BADENUM (EVOK_OBJ_NONE, an id out of range or not registered),
 * EVOK_E_BADSIZE (negative n_items, n_rows or item_stride_x, D <= 0, ldx < D, an instance whose n_items is neither 1 nor the
 * call's), EVOK_E_NOKERNEL, EVOK_E_NODATA (a registered id that declares data, not launched through an instance), EVOK_E_BADSIZE
 * (a data vector whose length is not D). */
int evok_eval_batched(int objective, const float* X, int64_t item_stride_x, int64_t ldx, int64_t n_items, int64_t n_rows, int64_t D,
                      uint64_t seed, uint64_t stream_id0, float* f, void* stream);
/* K2 of a transformed objective (evok_objective_register_transform) for a batch of populations: item b evaluates the n_rows rows of
 * X + b * item_stride_x (row pitch ldx) with y = M_b (x - o_b), M_b the row-major D x D matrix at M + b * item_stride_m (row pitch
 * D) and o_b the D-vector at o + b * item_stride_o (an item stride of 0 shares the operand), and writes f[b * n_rows ...].  Every
 * x_k - o_k is rounded to float32 before any product, so a row equal to o_b has y = 0 exactly.  Noise and data as in
 * evok_eval_batched: row r of item b draws on (seed, stream word stream_id0 + b) at global row r.  M and o are read in place.
 * The library picks the path from D (no option): up to D = 96, the crossover of the two paths timed on the H100 (DESIGN.md), one
 * fused launch per 65535
 * items computes y as one FP32 FMA chain per entry in increasing k and needs no workspace; above it each chunk of items (x - o
 * and y of a chunk within 256 MB) is three launches plus the GEMM's operand splits when M is not 16-byte aligned: x - o into
 * `ws`, y = (x - o) M^T by evok_gemm_nt_batched (3xTF32), and the fold of the x and y rows.  ws: at least
 * evok_eval_transform_workspace_bytes(M, item_stride_m, n_items, n_rows, D) bytes (0 on the fused path, where ws may be NULL).
 * Errors in this order: EVOK_E_NULLPTR (X, M, o, f), EVOK_E_BADENUM, EVOK_E_BADSIZE (negative counts or item strides, D <= 0,
 * ldx < D, an instance whose n_items is neither 1 nor the call's), EVOK_E_NOKERNEL (no transformed family), the data errors of
 * evok_eval_batched, EVOK_E_NULLPTR (ws NULL where the path needs one), EVOK_E_BADSIZE (ws_bytes too small). */
size_t evok_eval_transform_workspace_bytes(const float* M, int64_t item_stride_m, int64_t n_items, int64_t n_rows, int64_t D);
int evok_eval_transform_batched(int objective, const float* X, int64_t item_stride_x, int64_t ldx, const float* M, int64_t item_stride_m,
                                const float* o, int64_t item_stride_o, int64_t n_items, int64_t n_rows, int64_t D, uint64_t seed,
                                uint64_t stream_id0, void* ws, size_t ws_bytes, float* f, void* stream);
/* K3: f, w: [items][N].  ws: max(evok_rank_workspace_bytes(N), 8 * min(n_items, 65535) + 256) bytes */
int evok_rank_batched(int method, const float* f, int64_t N, int64_t n_items, int higher_is_better, float* w, void* ws, size_t ws_bytes,
                      void* stream);
int evok_elite_mask_batched(const float* w, int64_t N, int64_t n_items, int64_t num_elites, float* mask, void* ws, size_t ws_bytes, void* stream);
int evok_weights_adjust_batched(float* w, int64_t N, int64_t n_items, int mode, void* stream);
/* K4: X [items][n_rows][D] (item stride / row pitch given), w [items][n_rows], out_mu / out_sigma [items][D].  Errors in this order:
 * EVOK_E_NULLPTR, EVOK_E_BADENUM, EVOK_E_BADSIZE (negative counts or item strides, D <= 0, ldx < D), EVOK_E_ODDROWS,
 * EVOK_E_WORKSPACE. */
size_t evok_grad_batched_workspace_bytes(int64_t n_items, int64_t n_rows, int64_t D);
int evok_grad_batched(int form, const float* X, int64_t item_stride_x, int64_t ldx, const float* w, const float* mu, int64_t item_stride_mu,
                      const float* sigma, int64_t item_stride_sigma, int64_t n_items, int64_t n_rows, int64_t D, float scale_mu, float scale_sigma,
                      float* out_mu, float* out_sigma, void* ws, size_t ws_bytes, void* stream);
/* K4 over the population that evok_sample_eval_batched / evok_sample_batched drew from these mu and sigma with this (seed,
 * stream_id0), without reading it: every row with a non-zero weight is rebuilt from its Philox counters as
 * x = fmaf(sigma, z, mu) (item b on stream stream_id0 + b) and eps = x - mu, with the plan and workspace of evok_grad_batched.
 * The result is bit-identical to evok_grad_batched over the contiguous, 16-byte aligned X [items][n_rows][D] that the sampler
 * would have written.  Errors as evok_grad_batched. */
int evok_grad_batched_regen(int form, const float* w, const float* mu, int64_t item_stride_mu, const float* sigma, int64_t item_stride_sigma,
                            int64_t n_items, int64_t n_rows, int64_t D, uint64_t seed, uint64_t stream_id0, float scale_mu, float scale_sigma,
                            float* out_mu, float* out_sigma, void* ws, size_t ws_bytes, void* stream);
/* K5: g, velocity, center [items][D]; center += step.  sigma, g, lb / ub / mc vectors (nullable) [items][D] */
int evok_clipup_batched(const float* g, int64_t n_items, int64_t D, float* velocity, float* center, const float* stepsize_host,
                        const float* momentum_host, const float* max_speed_host, void* stream);
int evok_sigma_update_batched(float* sigma, const float* g, int64_t n_items, int64_t D, const float* lr_host, int exp_form, const float* lb_vec,
                              const float* ub_vec, const float* mc_vec, void* stream);

/* ---------------------------------------------------------------------------------------------
 * CMA-ES generation glue (algorithms/cmaes.py): the vector arithmetic between the dense contractions, fused.
 *   evok_cmaes_row_weights  : w_positive[i] = max(a_i, 0) (recombination weights, cmaes.py:468-475) and the active-CMA reweighting
 *       w_active[i] = a_i > 0 ? a_i : D * a_i / ||z_i||^2 (cmaes.py:531-535; active == 0: w_active = a).  One pass over Z.
 *   evok_cmaes_vector_update: one single-CTA kernel for update_m / update_p_sigma / update_sigma / _h_sig / update_p_c
 *       (cmaes.py:454-517, :31-46), all in place; k_out[0..2] = (c_mu, 1 - c1a - c_mu * sum(w), c1a * weighted_pc^2) are the
 *       coefficients of the covariance update for evok_gemm_nt_affine.  consts_host: 10 host floats
 *       (c_m, c_sigma, damp_sigma, c_c, c_1, c_mu, variance_discount_sigma, variance_discount_c, unbiased_expectation, sum(weights)).
 *       The generation counter of _h_sig comes from *steps_dev (then incremented by the kernel: CUDA-graph replay) or steps_host.
 * --------------------------------------------------------------------------------------------- */
int evok_cmaes_row_weights(const float* assigned_weights, const float* Z, int64_t ldz, int64_t N, int64_t D, int active, float* w_positive,
                           float* w_active, void* stream);
int evok_cmaes_vector_update(const float* local_disp, const float* shaped_disp, int64_t D, float* m, float* p_sigma, float* p_c, float* sigma_dev,
                             int64_t* steps_dev, int64_t steps_host, const float* consts_host, int csa_squared, float* k_out, float* h_sig_out,
                             void* stream);
/* The same two stages for n_items independent searches (functional CMA-ES), per item the bits of the single call:
 *   evok_rank_table_batched        : keys, out [items][N], one shared table; the workspace of evok_rank_table.
 *   evok_cmaes_row_weights_batched : Z_b at Z + b * item_stride_z (pitch ldz); assigned_weights, w_positive, w_active [items][N].
 *   evok_cmaes_vector_update_batched: one CTA per item; local_disp, shaped_disp, m, p_sigma, p_c [items][D], sigma_dev [items],
 *       k_out [items][3]; the constants and the generation counter steps_host are shared.
 *   evok_cmaes_vector_update_batched_steps: the same with one generation counter per item: item b's _h_sig reads steps_dev[b]
 *       (int64, device) and the kernel increments it, as the single call does with its steps_dev.  Errors: those of
 *       evok_cmaes_vector_update_batched, and EVOK_E_NULLPTR for steps_dev. */
int evok_rank_table_batched(const float* keys, int64_t N, int64_t n_items, int descending, const float* table, float* out, void* ws, size_t ws_bytes,
                            void* stream);
int evok_cmaes_row_weights_batched(const float* assigned_weights, const float* Z, int64_t item_stride_z, int64_t ldz, int64_t n_items, int64_t N,
                                   int64_t D, int active, float* w_positive, float* w_active, void* stream);
int evok_cmaes_vector_update_batched(const float* local_disp, const float* shaped_disp, int64_t n_items, int64_t D, float* m, float* p_sigma,
                                     float* p_c, float* sigma_dev, int64_t steps_host, const float* consts_host, int csa_squared, float* k_out,
                                     void* stream);
int evok_cmaes_vector_update_batched_steps(const float* local_disp, const float* shaped_disp, int64_t n_items, int64_t D, float* m,
                                           float* p_sigma, float* p_c, float* sigma_dev, int64_t* steps_dev, const float* consts_host,
                                           int csa_squared, float* k_out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Separable CMA-ES (diagonal C, algorithms/cmaes.py with separable=True) as three kernels plus evok_rank_table, with no host
 * reads.  With s = sigma * A (the per-column stdev of the sampler) one generation is
 *   evok_sample_eval_sq : x_i = fmaf(s, z_i, m) (X nullable: lazy population), f_i = objective(x_i), q_i = ||z_i||^2
 *   evok_rank_table     : aw = weights[rank(f)]
 *   evok_sepcma_moments : regenerates z_i from Philox and reduces local = sum_i a_i z_i, S2 = sum_i b_i z_i^2, wsum = sum_i b_i with
 *                         a_i = max(aw_i, 0), b_i = active ? (aw_i > 0 ? aw_i : D aw_i / q_i) : aw_i   (cmaes.py:454-481, :519-535);
 *                         rows with a_i = b_i = 0 are not regenerated (their q_i is not read).  Fixed summation order, no atomics.
 *   evok_sepcma_update  : m, p_sigma, sigma, h_sig, p_c (the arithmetic of evok_cmaes_vector_update, with shaped = A * local), then
 *                         C <- C + c1a (p_c^2 - C) + c_mu (A^2 S2 - wsum C) (cmaes.py:536-545, separable branch), the stdev bounds
 *                         with the new sigma (cmaes.py:49-79; NaN = no bound), A <- sqrt(C) when (steps + 1) % decompose_C_freq == 0,
 *                         s <- sigma A.  One CTA.  m_prev / s_prev (nullable) receive m and s before the update: the centre and stdev
 *                         the population of this generation was drawn from.  Step counter as in evok_cmaes_vector_update.
 * --------------------------------------------------------------------------------------------- */
/* evok_sample_eval for a non-symmetric population that also writes q[i] = sum_j z_ij^2 of the unscaled normals.  X and f are
 * bit-identical to evok_sample_eval with the same arguments.  objective may be EVOK_OBJ_NONE only when X is given. */
int evok_sample_eval_sq(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows, int64_t D,
                        uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev, float* f, float* q, void* stream);
size_t evok_sepcma_workspace_bytes(int64_t n_rows, int64_t D);
/* aw: the n_rows assigned weights; q: nullable when active == 0; (seed, stream_id, stream_offset_dev, row0) as for the sampler */
int evok_sepcma_moments(const float* aw, const float* q, int active, int64_t row0, int64_t n_rows, int64_t D, uint64_t seed, uint64_t stream_id,
                        const uint32_t* stream_offset_dev, float* local, float* S2, float* wsum, void* ws, size_t ws_bytes, void* stream);
/* consts_host: the 10 floats of evok_cmaes_vector_update (the last one, sum(weights), is not used: wsum comes from the device) */
int evok_sepcma_update(const float* local, const float* S2, const float* wsum, int64_t D, float* m, float* p_sigma, float* p_c, float* sigma_dev,
                       float* C, float* A, float* s, float* m_prev, float* s_prev, int64_t* steps_dev, int64_t steps_host, const float* consts_host,
                       int csa_squared, int64_t decompose_C_freq, float stdev_min, float stdev_max, float* h_sig_out, void* stream);
/* The same two stages for n_items independent separable searches (functional separable CMA-ES), whose populations may have been
 * repaired or replaced after the ask, so the steps are recovered from the rows: z_ij = (x_ij - m_j) / s_j (correctly rounded) and
 * q_i = ||z_i||^2 of that z.
 *   evok_sepcma_moments_batched: local = sum_i a_i z_i, S2 = sum_i b_i z_i^2, wsum = sum_i b_i per item, with the weights of
 *       evok_sepcma_moments (b_i = D aw_i / q_i for the negative weights when active).  X: [items][n_rows][D] at item stride
 *       item_stride_x and row pitch ldx; NULL: the rows with a non-zero weight are rebuilt as the batched sampler stored them from
 *       (seed, stream_id0 + b), x = fmaf(s, z, m), with the same bits as the stored rows.  m, s, local, S2 [items][D]; aw [items][n_rows];
 *       wsum [items].  A row pass writes q of the rows with a negative weight to the workspace (active only), then the column pass
 *       reduces: the population is read (or rebuilt) at most twice, rows of zero weight not at all.  Fixed summation order, no
 *       atomics; item b gives the bits of a one-item call on its operands with stream_id0 + b.  Errors in this order:
 *       EVOK_E_NULLPTR, EVOK_E_BADSIZE (n_items < 0, n_rows <= 0, D <= 0, with X: ldx < D or a negative item stride),
 *       EVOK_E_WORKSPACE (none with n_items == 0).
 *   evok_sepcma_update_batched: evok_sepcma_update with one CTA per item, per item the bits of the single call; local, S2, m, p_sigma,
 *       p_c, C, A, s [items][D], wsum, sigma_dev [items].  The constants, the generation counter and the stdev bounds are shared.
 *   evok_sepcma_update_batched_steps: the same with one generation counter per item, steps_dev[b] (int64, device, incremented by
 *       the kernel): item b's _h_sig and its decomposition schedule, (steps_dev[b] + 1) % decompose_C_freq == 0, follow its own
 *       counter.  Errors: those of evok_sepcma_update_batched, and EVOK_E_NULLPTR for steps_dev. */
size_t evok_sepcma_moments_batched_workspace_bytes(int64_t n_items, int64_t n_rows, int64_t D);
int evok_sepcma_moments_batched(const float* X, int64_t item_stride_x, int64_t ldx, const float* m, const float* s, const float* aw, int active,
                                int64_t n_items, int64_t n_rows, int64_t D, uint64_t seed, uint64_t stream_id0, float* local, float* S2, float* wsum,
                                void* ws, size_t ws_bytes, void* stream);
int evok_sepcma_update_batched(const float* local, const float* S2, const float* wsum, int64_t n_items, int64_t D, float* m, float* p_sigma, float* p_c,
                               float* sigma_dev, float* C, float* A, float* s, int64_t steps_host, const float* consts_host, int csa_squared,
                               int64_t decompose_C_freq, float stdev_min, float stdev_max, void* stream);
int evok_sepcma_update_batched_steps(const float* local, const float* S2, const float* wsum, int64_t n_items, int64_t D, float* m, float* p_sigma,
                                     float* p_c, float* sigma_dev, float* C, float* A, float* s, int64_t* steps_dev, const float* consts_host,
                                     int csa_squared, int64_t decompose_C_freq, float stdev_min, float stdev_max, void* stream);

/* Restarts of the functional CMA-ES families: the stage after a batched update (evok_cmaes_vector_update_batched_steps + the
 * covariance update + Cholesky, or evok_sepcma_update_batched_steps), one CTA per item, no host reads.
 *   evok_cma_restart_batched: per item b, with N = n_rows and g = item_steps[b] (the generations since the item's (re)start, the
 *       update already counted),
 *       - best ever: the best finite f of this generation (under `maximize`; the lower row on ties), if strictly better than
 *         best_f[b], goes to best_f[b] and its row to best_x[b] (D floats): row i of X, or with X == NULL (separable only) the
 *         row the batched sampler stored for (draw_seed, stream b, row i), x = fmaf(s_draw, z, m_draw), the same bits;
 *       - history [items][H]: slot (g - 1) % H <- that best value (NaN when no f was finite);
 *       - stop_flags[b] (int32) <- the criteria that fire, thresholds_host[0..5] (6 host floats, NaN = off):
 *           bit 0 tol_fun    g >= H and max - min over the H history slots and the N values of f < thresholds[0] (all finite)
 *           bit 1 tol_x      sigma max_j max(|p_c,j|, sqrt(C_jj)) < thresholds[1] sigma0[b]
 *           bit 2 tol_x_up   sigma max_j sqrt(C_jj) > thresholds[2] sigma0[b]
 *           bit 3 max_cond   full: (max_j A_jj / min_j A_jj)^2 > thresholds[3]; every Cholesky pivot A_jj^2 lies in
 *                            [lambda_min(C), lambda_max(C)], so this is a lower bound of cond(C) and never fires early;
 *                            separable: max_j C_j / min_j C_j > thresholds[3]
 *           bit 4 min_fitness_stdev  the unbiased standard deviation of the N values (N > 1, finite) < thresholds[4]
 *           bit 5 max_generations    g >= thresholds[5]
 *           bit 6 non-finite (always on)  sigma <= 0, or sigma, an entry of m, p_sigma, p_c or diag C is not finite
 *           bit 7 small-run budget (BIPOP only, evok_cma_restart_batched_bipop; never set by this entry)
 *       - an item with a flag restarts: m_j = lb_j + (ub_j - lb_j) u_j (float32, unfused) with u_j = uniform24 of word j & 3 of
 *         Philox4x32-10(counter (j >> 2, 0, 0xFF000000, stream word b), key (seed, stream 0)) -- no sample counter (third word
 *         below 2^31) or noise counter (0x80.. to 0x87..) has this third word; sigma <- sigma0[b], p_sigma = p_c = 0,
 *         item_steps[b] = 0, history row NaN, num_restarts[b] (int64) += 1; C = A = I (full: a second, grid-wide launch masked by
 *         the flags), separable: C = A = 1 and s = sigma0[b].
 *       separable != 0: C, A, s [items][D]; else C, A [items][D][D] (s unused, nullable).  m, p_sigma, p_c, best_x, m_draw,
 *       s_draw [items][D]; f [items][N]; X at item_stride_x / ldx; sigma, sigma0, best_f [items]; lb, ub at item_stride_bounds
 *       (0: shared, or D).  One launch (separable) or two (full).  Errors in this order: EVOK_E_NULLPTR (any state pointer,
 *       thresholds_host, X for the full family, s for the separable one, m_draw / s_draw without X), EVOK_E_BADSIZE (n_items < 0,
 *       n_rows <= 0, D <= 0, H <= 0, with X: ldx < D or a negative item stride, item_stride_bounds not 0 or D).  Nothing is
 *       launched for n_items == 0. */
int evok_cma_restart_batched(int separable, const float* f, const float* X, int64_t item_stride_x, int64_t ldx, const float* m_draw,
                             const float* s_draw, uint64_t draw_seed, int64_t n_items, int64_t n_rows, int64_t D, int maximize, int64_t* item_steps,
                             float* m, float* sigma, float* p_sigma, float* p_c, float* C, float* A, float* s, float* history, int64_t H,
                             float* best_x, float* best_f, int64_t* num_restarts, int32_t* stop_flags, const float* sigma0, const float* lb,
                             const float* ub, int64_t item_stride_bounds, const float* thresholds_host, uint64_t seed, void* stream);

/* IPOP restarts (padded populations): every item draws N = max_popsize rows, and item b uses only its first n_b rows, n_b =
 * counts[tier[b]] of a ladder of population sizes, with the constants of its tier.  tier [items] int32 and the tables (counts [K]
 * int32 with 1 <= counts[k] <= N, tables [K][N], consts_dev [K][10], decompose_C_freq_dev [K] int64 >= 1, tier_history [K] int64
 * with 1 <= tier_history[k] <= H) are device memory; nothing is read back.  Rows n_b..N-1 of item b are pad rows: whatever their
 * keys, values or Z hold (NaN and inf included), they reach no output but their own zero weights.
 *   evok_rank_table_batched_tiered: item b ranks its first n_b keys (the counting rank of evok_rank_table_batched, stable, NaN the
 *       largest) and writes tables[tier[b]][position] to them, 0 to its pad rows; an item with n_b = N gets the bits of
 *       evok_rank_table_batched with table row tier[b].  No workspace.  Errors: EVOK_E_NULLPTR, EVOK_E_BADSIZE (N < 0, N > 8192,
 *       n_items < 0).  Grid y = item, chunks of 65535 items.
 *   evok_cmaes_row_weights_batched_tiered: evok_cmaes_row_weights_batched on the first n_b rows of item b, w_positive = w_active =
 *       0 on its pad rows.  Errors: EVOK_E_NULLPTR (tier, counts first), then those of evok_cmaes_row_weights_batched.
 *   evok_cmaes_vector_update_batched_tiered: evok_cmaes_vector_update_batched_steps with item b's constants read from row tier[b]
 *       of consts_dev (the 10 floats of consts_host; its weights_sum enters k_out).  Errors: EVOK_E_NULLPTR (steps_dev, tier,
 *       consts_dev and the state), EVOK_E_BADSIZE (n_items < 0, D <= 0).
 *   evok_sepcma_update_batched_tiered: evok_sepcma_update_batched_steps with item b's constants from row tier[b] of consts_dev and
 *       its decomposition schedule (steps_dev[b] + 1) % decompose_C_freq_dev[tier[b]] == 0.  Errors: EVOK_E_NULLPTR (steps_dev,
 *       tier, consts_dev, decompose_C_freq_dev and the state), EVOK_E_BADSIZE (n_items < 0, D <= 0).
 *   evok_cma_restart_batched_tiered: evok_cma_restart_batched (n_rows = N, H the ring length of every history row) with, for
 *       item b, N = counts[tier[b]] (tier_counts) and H = tier_history[tier[b]]: the best row, the history slot (g - 1) % H, the
 *       tol_fun and min_fitness_stdev criteria use only the first N values or rows and the first H slots (a lazy separable row
 *       is rebuilt only for the best of those N).  Then num_evaluations[b] (int64) += N, and a restarted item moves to tier
 *       min(tier[b] + 1, n_tiers - 1) and has its whole history row set to NaN.  Errors: those of evok_cma_restart_batched in its
 *       order, with EVOK_E_NULLPTR also for tier, tier_counts, tier_history and num_evaluations, and EVOK_E_BADSIZE also for
 *       n_tiers < 1. */
int evok_rank_table_batched_tiered(const float* keys, int64_t N, int64_t n_items, int descending, const float* tables, const int32_t* tier,
                                   const int32_t* counts, float* out, void* stream);
int evok_cmaes_row_weights_batched_tiered(const float* assigned_weights, const float* Z, int64_t item_stride_z, int64_t ldz, int64_t n_items,
                                          int64_t N, int64_t D, int active, const int32_t* tier, const int32_t* counts, float* w_positive,
                                          float* w_active, void* stream);
int evok_cmaes_vector_update_batched_tiered(const float* local_disp, const float* shaped_disp, int64_t n_items, int64_t D, float* m,
                                            float* p_sigma, float* p_c, float* sigma_dev, int64_t* steps_dev, const int32_t* tier,
                                            const float* consts_dev, int csa_squared, float* k_out, void* stream);
int evok_sepcma_update_batched_tiered(const float* local, const float* S2, const float* wsum, int64_t n_items, int64_t D, float* m, float* p_sigma,
                                      float* p_c, float* sigma_dev, float* C, float* A, float* s, int64_t* steps_dev, const int32_t* tier,
                                      const float* consts_dev, const int64_t* decompose_C_freq_dev, int csa_squared, float stdev_min,
                                      float stdev_max, void* stream);
int evok_cma_restart_batched_tiered(int separable, const float* f, const float* X, int64_t item_stride_x, int64_t ldx, const float* m_draw,
                                    const float* s_draw, uint64_t draw_seed, int64_t n_items, int64_t n_rows, int64_t D, int maximize,
                                    int64_t* item_steps, float* m, float* sigma, float* p_sigma, float* p_c, float* C, float* A, float* s,
                                    float* history, int64_t H, float* best_x, float* best_f, int64_t* num_restarts, int32_t* stop_flags,
                                    const float* sigma0, const float* lb, const float* ub, int64_t item_stride_bounds,
                                    const float* thresholds_host, uint64_t seed, int32_t* tier, const int32_t* tier_counts,
                                    const int64_t* tier_history, int64_t n_tiers, int64_t* num_evaluations, void* stream);

/* BIPOP restarts (Hansen, GECCO 2009 workshops): IPOP's padded populations with two regimes per item, large runs that climb the
 * ladder and small runs of random population size and step size, each given a similar share of the evaluations.
 *   evok_cma_restart_batched_bipop: evok_cma_restart_batched_tiered (sigma0 renamed sigma_def: the default step size per item)
 *       with a per-item policy in place of the tier advance.  Tiers 0..n_large-1 of the tables are the ladder lambda_0 =
 *       popsize0 .. lambda_{K-1}; tier n_large + (lambda - popsize0) is a small run of population size lambda, for every lambda in
 *       [popsize0, max(popsize0, floor(lambda_{K-1} / 2))], so n_tiers is at least n_large + 1.  Per item b, device memory:
 *       regime [items] int32 (0 the first run, 1 a large run, 2 a small run), large_tier [items] int32 (l: the rung of the latest
 *       large run, 0 before any), large_evaluations, small_evaluations, last_large_evaluations [items] int64 (n_L, n_S, n_last),
 *       run_stdev [items] float (the step size the current run started with).  With N = counts[tier[b]] and g = item_steps[b]:
 *       - n_L (regime 1) or n_S (regime 2) grows by N; the first run counts in neither;
 *       - tol_x and tol_x_up compare against run_stdev[b] instead of sigma0;
 *           bit 7 small-run budget  regime 2 and 2 g N >= n_last (the run has used half the evaluations of the latest large run)
 *       - an item with a flag: if its run was large, n_last <- g N.  Then the next run is large when n_L <= n_S (so the first
 *         restart is): l <- min(l + 1, n_large - 1), tier = l, run_stdev = sigma_def.  Otherwise small: u1, u2 = uniform24 of
 *         words x and y of Philox4x32-10(counter (0, 1, 0xFF000000, stream word b), key (seed, stream 0)) -- the reset centres
 *         have second word 0, so no other draw has this counter; lambda_s = max(popsize0, floor(popsize0 exp(u1^2 log(0.5
 *         counts[l] / popsize0)))) and run_stdev = (float)(sigma_def 10^(-2 u2)), both in float64; tier = n_large + lambda_s -
 *         popsize0 (at most n_tiers - 1).  The reset is evok_cma_restart_batched's with run_stdev[b] in place of sigma0[b]
 *         (sigma, and s for the separable family).
 *       Errors: those of evok_cma_restart_batched_tiered in its order, with EVOK_E_NULLPTR also for regime, large_tier, the three
 *       budgets and run_stdev, and EVOK_E_BADSIZE also for n_large < 1, n_large >= n_tiers, popsize0 < 1. */
int evok_cma_restart_batched_bipop(int separable, const float* f, const float* X, int64_t item_stride_x, int64_t ldx, const float* m_draw,
                                   const float* s_draw, uint64_t draw_seed, int64_t n_items, int64_t n_rows, int64_t D, int maximize,
                                   int64_t* item_steps, float* m, float* sigma, float* p_sigma, float* p_c, float* C, float* A, float* s,
                                   float* history, int64_t H, float* best_x, float* best_f, int64_t* num_restarts, int32_t* stop_flags,
                                   const float* sigma_def, const float* lb, const float* ub, int64_t item_stride_bounds,
                                   const float* thresholds_host, uint64_t seed, int32_t* tier, const int32_t* tier_counts,
                                   const int64_t* tier_history, int64_t n_tiers, int64_t* num_evaluations, int32_t* regime, int32_t* large_tier,
                                   int64_t* large_evaluations, int64_t* small_evaluations, int64_t* last_large_evaluations, float* run_stdev,
                                   int64_t n_large, int64_t popsize0, void* stream);

/* Cholesky factorisation A = L L^T (fp32, lower; the strictly upper part of L is zeroed, like torch.linalg.cholesky).  Replaces
 * CMAES.decompose_C (cmaes.py:555-565, torch.linalg.cholesky -> cuSOLVER potrf).  ONE persistent kernel: 64 x 64 tiles, left-looking
 * tile dataflow with per-tile release / acquire flags instead of a launch (or grid barrier) per panel step.  Only the lower triangle
 * of A is read.  L must not alias A.  A matrix that is not positive definite yields NaNs (no error code: nothing is read back). */
size_t evok_cholesky_workspace_bytes(int64_t n);
int evok_cholesky(const float* A, int64_t lda, int64_t n, float* L, int64_t ldl, void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Peer exchange over NVLink / NVSwitch: the two collectives of the sharded generation (the reference's Ray round trip,
 * core.py:2762-3073 + algorithms/distributed/gaussian.py:199-272; evotorch_b200/distributed.py) fused into their
 * producing kernels.  One process per GPU; every rank owns one "exchange buffer" that all peers map (CUDA IPC).
 *
 *   evok_peer_alloc / open / close / free : the only entry points that allocate.  `handle` is a 64-byte cudaIpcMemHandle_t
 *       to be passed to the other processes (any transport).  The buffer is zero-filled.
 *   evok_sample_eval_push : evok_sample_eval whose fitness store goes to row (row0 + i) of EVERY peer's fitness vector
 *       (peer_f_host[p] = base of peer p's N-float vector; the *_host tables are host arrays of `world` device pointers) -- the all-gather.  The last CTA raises flag[rank] = *epoch_dev + 1 in
 *       every peer's flag array (peer_flags_host[p] = base of peer p's `world` 64-bit flags).
 *   evok_peer_wait : one warp spins until all `world` local flags reach *epoch_dev + 1, then advances *epoch_dev.  After
 *       `timeout_ns` it gives up, sets *err_dev = 1 and advances anyway (no hang; the host checks err_dev when it likes).
 *   evok_grad_push : evok_grad / evok_grad_regen (X == NULL) whose finalisation writes this rank's (grad_mu | grad_sigma)
 *       into slot `rank` of every peer's slot array (peer_slots_host[p] = base of world x 2D floats) and raises the flags.
 *   evok_peer_reduce : waits like evok_peer_wait, then out[j] = sum over ranks (in rank order: bit-identical on every GPU)
 *       of slots[r * n + j] -- the all-reduce.
 * `done_dev` is a zero-initialised local uint32 per exchange point; `epoch_dev` a zero-initialised local uint64 per
 * exchange point.  Everything is stream-ordered and CUDA-graph capturable (the pointers are baked into the launch).
 * --------------------------------------------------------------------------------------------- */
/* Sharded ranking (round 2): the fitness all-gather + replicated global sort of the sharded generation replaced by a LOCAL
 * sort + an exchange of sorted keys.  Each GPU sorts only its own n_local fitnesses (stable LSD radix, 8 launches), pushes the
 * sorted orderable keys into every peer's key table (peer_keys_host[p] = base of peer p's N-entry uint32 table) together with
 * its local fitness sum (peer_fsum_host[p] = base of peer p's `world` doubles) and raises its flag; then, after all flags have
 * arrived, every local row finds its GLOBAL position = local position + sum over the other shards of the number of their keys
 * that precede it (binary searches over the L2-resident table; ties by global index exactly like the global stable sort) and
 * writes its utility.  Replaces, per GPU, tools/ranking.py:24-124 on the all-gathered vector (the Ray path ranks per actor,
 * core.py:3289).  Results are bit-identical to evok_rank on the gathered vector; methods: CENTERED, LINEAR, NES.
 * row_offsets_host: world + 1 global row offsets of the shards (host array); w_local: n_local utilities in local row order;
 * mean_out (nullable): global mean fitness.  done_dev: THREE zero-initialised uint32; ws: evok_rank_workspace_bytes(n_local). */
int evok_rank_sharded(int method, const float* f_local, int64_t N, int higher_is_better, int world, int rank,
                      const int64_t* row_offsets_host, void* const* peer_keys_host, void* const* peer_fsum_host,
                      void* const* peer_flags_host, uint64_t* epoch_dev, uint32_t* done_dev, uint32_t* err_dev, uint64_t timeout_ns,
                      float* w_local, float* mean_out, void* ws, size_t ws_bytes, void* stream);

int evok_peer_alloc(size_t bytes, void** dev_ptr_out_host, void* handle_out_64B_host);
int evok_peer_open(const void* handle_64B_host, void** dev_ptr_out_host);
int evok_peer_close(void* dev_ptr);
int evok_peer_free(void* dev_ptr);
int evok_sample_eval_push(int objective, float* X, int64_t ldx, const float* mu, const float* sigma, int64_t row0, int64_t n_rows,
                          int64_t D, int symmetric, uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev, int world,
                          int rank, void* const* peer_f_host, void* const* peer_flags_host, const uint64_t* epoch_dev, uint32_t* done_dev,
                          void* stream);
/* evok_peer_push: the all-gather as ONE small kernel behind the producer: CTA p copies this rank's slice (n_bytes at src_local) to
 * offset dst_offset_bytes of peer p's buffer (peer_base_host[p]) with 16-byte stores, fences once and raises flag[rank] = *epoch_dev + 1
 * on that peer.  Consumer: evok_peer_wait, as for evok_sample_eval_push. */
int evok_peer_push(const void* src_local, int64_t n_bytes, int64_t dst_offset_bytes, int world, int rank, void* const* peer_base_host,
                   void* const* peer_flags_host, const uint64_t* epoch_dev, void* stream);
int evok_peer_wait(const uint64_t* flags_local, int world, uint64_t* epoch_dev, uint32_t* err_dev, uint64_t timeout_ns, void* stream);
int evok_grad_push(int form, const float* X, int64_t ldx, const float* w, const float* mu, const float* sigma, int64_t row0,
                   int64_t n_rows, int64_t D, uint64_t seed, uint64_t stream_id, const uint32_t* stream_offset_dev, float scale_mu,
                   float scale_sigma, int world, int rank, void* const* peer_slots_host, void* const* peer_flags_host,
                   const uint64_t* epoch_dev, uint32_t* done_dev, void* ws, size_t ws_bytes, void* stream);
int evok_peer_reduce(const float* slots_local, int world, int64_t n, const uint64_t* flags_local, uint64_t* epoch_dev,
                     uint32_t* done_dev, uint32_t* err_dev, uint64_t timeout_ns, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Limited-memory matrix adaptation (LM-MA-ES, Loshchilov, Glasmachers & Beyer, IEEE TEVC 23(2), 2019) for n_items independent
 * searches (functional LM-MA-ES).  Item b holds y [D], sigma, p_sigma [D], m vectors M [m][D] and G = M M^T [m][m]; all operands
 * are contiguous [items][...].  k = min(t, m) is the number of vectors in use at generation t.  consts_host: 2 + 2m doubles,
 * (c_sigma, mu_eff, c_d,1 .. c_d,m, c_c,1 .. c_c,m).  Limits: 2 <= n_rows <= EVOK_LMMAES_MAX_POPSIZE, 1 <= m <=
 * EVOK_LMMAES_MAX_VECTORS, 0 <= k <= m.  Column passes take tiles of 512 columns whatever n_items, so item b gives the bits of a
 * one-item call on its own operands; sums are in fixed order, with no atomics.  Each entry launches per item chunk of at most
 * 65535 items, one after another.  The workspace holds one chunk.
 *   evok_lmmaes_ask_batched: X [items][n_rows][D], x_i = y + sigma d_i, d_i = z_i after k steps d <- (1 - c_d,j) d + c_d,j M_j (M_j^T d),
 *       in the coefficient form: P = M_k Z^T (a Gram pass over z rebuilt from Philox), the recursion for beta (one CTA per item),
 *       and the pass that writes x = y + sigma (alpha z + beta M_k).  z_i of item b is the row the batched sampler draws with
 *       (seed, stream_id0 + b).  With k = 0 only the write pass runs, and x = fmaf(sigma, z, y): the bits of evok_sample_batched
 *       with mean y and stdev sigma.  Launches per chunk: 3, or 1 with k = 0.
 *   evok_lmmaes_tell_batched: aw [items][n_rows], the weights of the rows' ranks (0 for rows outside the best mu).  The rows with a
 *       non-zero weight are read once: d = (x - y) / sigma, S_d = sum w_i d_i and Q = M_k D^T; the recovery of z (one CTA per
 *       item) gives S_z = a S_d + sum_j c_j M_j; then M_j' = (1 - c_c,j) M_j + sqrt(mu_eff c_c,j (2 - c_c,j)) S_z for every j < m,
 *       p_sigma' = (1 - c_sigma) p_sigma + sqrt(mu_eff c_sigma (2 - c_sigma)) S_z, y' = y + sigma S_d, G' = M' M'^T of the M' written,
 *       sigma' = sigma exp((c_sigma / 2)(|p_sigma'|^2 / D - 1)).  The outputs must not overlap the inputs.  Launches per chunk: 4.
 * Errors in this order: EVOK_E_NULLPTR, EVOK_E_BADSIZE (a count outside its limits), EVOK_E_WORKSPACE.
 * --------------------------------------------------------------------------------------------- */
#define EVOK_LMMAES_MAX_VECTORS 64
#define EVOK_LMMAES_MAX_POPSIZE 128
size_t evok_lmmaes_workspace_bytes(int64_t n_items, int64_t n_rows, int64_t D, int64_t m);
int evok_lmmaes_ask_batched(float* X, const float* y, const float* sigma, const float* M, const float* G, int64_t n_items, int64_t n_rows,
                            int64_t D, int64_t m, int64_t k, const double* consts_host, uint64_t seed, uint64_t stream_id0, void* ws,
                            size_t ws_bytes, void* stream);
int evok_lmmaes_tell_batched(const float* X, const float* aw, const float* y, const float* sigma, const float* p_sigma, const float* M,
                             const float* G, int64_t n_items, int64_t n_rows, int64_t D, int64_t m, int64_t k, const double* consts_host,
                             float* y_out, float* sigma_out, float* p_sigma_out, float* M_out, float* G_out, void* ws, size_t ws_bytes,
                             void* stream);

/* ---------------------------------------------------------------------------------------------
 * Functional XNES (csrc/evok_xnes.cu): one CTA per item, the working matrices in shared memory, 1 <= D <= EVOK_XNES_MAX_D.
 * Items go in chunks of at most 65535, one launch each; sums are in fixed order, with no atomics, so item b gives the bits of a
 * one-item call on its own operands.
 *   evok_sym_expm_pair_batched: for every symmetric S [items][D][D], F_plus = expm(S) - I and F_minus = expm(-S) - I (the expm1
 *       form keeps the relative precision of a tiny S).  Scaling and squaring with s = max(0, ceil(log2 |S|_1)) per item, a
 *       degree-11 Taylor core in S^2 / 4^s shared by both signs, and F <- 2F + F^2 s times for each sign.
 *   evok_xnes_tell_batched: X [items][n_rows][D], w [items][n_rows] the utilities (already centred where the ranking needs it),
 *       mu [items][D], A and A_inv [items][D][D].  z_r = A_inv (x_r - mu) for the rows with w_r != 0, d = sum w_r z_r,
 *       S = (lr_A / 2)(sum w_r z_r z_r^T - (sum w_r) I), then mu' = mu + A (lr_mu d), A' = A + A F+, A_inv' = A_inv + F- A_inv with
 *       the exponential pair of S.  The outputs must not overlap the inputs.
 * Errors in this order: EVOK_E_NULLPTR, EVOK_E_BADSIZE (n_items < 0, D < 1, D > EVOK_XNES_MAX_D, n_rows < 2).
 * --------------------------------------------------------------------------------------------- */
#define EVOK_XNES_MAX_D 96
int evok_sym_expm_pair_batched(const float* S, int64_t n_items, int64_t D, float* F_plus, float* F_minus, void* stream);
int evok_xnes_tell_batched(const float* X, const float* w, const float* mu, const float* A, const float* A_inv, int64_t n_items, int64_t n_rows,
                           int64_t D, float lr_mu, float lr_A, float* mu_out, float* A_out, float* A_inv_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EVOK_H_ */
