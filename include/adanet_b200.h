/*
 * adanet_b200.h -- C ABI of the H100-native AdaNet candidate-training engine.
 *
 * The reference (tensorflow/adanet v0.9.0) has NO FFI boundary: its hot path is
 * Python that builds a TF1 graph, executed by TensorFlow's stock CPU kernels
 * (SURVEY.md section 8b).  These entry points are therefore *new*; each one
 * names the reference code whose per-step arithmetic it replaces
 * (file:line relative to tensorflow/adanet v0.9.0).  INTEGRATION.md shows the ctypes
 * binding a reference maintainer would add.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless
 *     its name ends in _host; the caller (PyTorch) owns every buffer;
 *   - all work is enqueued on the caller-supplied cudaStream_t (passed as
 *     void*); no call synchronises the device or allocates device memory;
 *   - all matrices are dense row-major fp32; labels are int64;
 *   - returns 0 on success, negative errno-style code otherwise, and
 *     adn_last_error() returns a thread-local human-readable message;
 *   - re-entrant across streams; the only process-global state is a cache of
 *     TMA descriptors keyed by (plane pointer, rows, k-blocks, majorness, format)
 *     (csrc/planes.cu make_map), kernel attributes, and the two process-wide
 *     settings adn_set_dense_path / adn_set_plane_format.
 *   - reductions (loss means, bias/weight gradients) use a fixed summation
 *     order: results are run-to-run deterministic.
 */
#ifndef ADANET_B200_H_
#define ADANET_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ADN_OK 0
#define ADN_ERR_INVALID (-22)     /* EINVAL: bad shape / null pointer / bad enum */
#define ADN_ERR_CUDA (-5)         /* EIO: a CUDA runtime/driver call failed     */
#define ADN_ERR_UNSUPPORTED (-95) /* EOPNOTSUPP: shape not supported by a path  */
#define ADN_ERR_WORKSPACE (-12)   /* ENOMEM: caller workspace too small         */

/* activation fused into adn_dense_fwd (simple_dnn.py:72-78 uses relu) */
#define ADN_ACT_NONE 0
#define ADN_ACT_RELU 1

/* head / loss kinds  [TF heads called at adanet/core/ensemble_builder.py:571-583] */
#define ADN_HEAD_SOFTMAX_XENT 0 /* MultiClassHead: mean sparse softmax-CE      */
#define ADN_HEAD_MSE 1          /* RegressionHead: mean squared error          */
#define ADN_HEAD_SIGMOID_XENT 2 /* BinaryClassHead: mean sigmoid-CE            */

/* mixture weight types: adanet/ensemble/weighted.py:139-147 */
#define ADN_MIX_SCALAR 0
#define ADN_MIX_VECTOR 1
#define ADN_MIX_MATRIX 2 /* members arrive already multiplied by their matrix */

/* optimizers (TF1 update rules; call sites simple_dnn.py:110, weighted.py:616) */
#define ADN_OPT_SGD 0
#define ADN_OPT_MOMENTUM 1
#define ADN_OPT_RMSPROP 2
#define ADN_OPT_ADAM 3
/* Momentum whose learning rate follows tf.train.cosine_decay(lr, step, decay_steps, alpha) of the per-optimizer
 * step counter (SimpleCNNBuilder.build_subnetwork_train_op, customizing_adanet.ipynb): hyper = {lr, momentum,
 * decay_steps, alpha}; lr_t = lr * ((1-alpha) * 0.5 * (1 + cos(pi * min(step, decay_steps) / decay_steps)) + alpha) */
#define ADN_OPT_MOMENTUM_COSINE 4

/* compute paths for the dense kernels (adn_set_dense_path / adn_query) */
#define ADN_PATH_AUTO 0    /* tensor-core split-plane GEMM where shapes allow, SIMT fp32 otherwise */
#define ADN_PATH_SIMT 1    /* CUDA-core fp32 FMA everywhere                         */
#define ADN_PATH_TCGEN05 2 /* force tensor path; unsupported shapes return an error  */

/* split-plane formats of the tensor-core dense pipeline (adn_set_plane_format; csrc/plane_fmt.cuh) */
#define ADN_PLANES_TF32 0 /* hi/lo TF32, 4 B per value, tf32 MMAs, fp32 exponent range                 */
#define ADN_PLANES_F16 1  /* hi/lo' fp16 (lo' carries 2^11), 2 B per value, fp16 MMAs (default)         */

/* adn_query keys */
#define ADN_Q_VERSION 0
#define ADN_Q_DENSE_BWD_WORKSPACE_BYTES 1 /* a=batch b=in c=out */
#define ADN_Q_HEAD_WORKSPACE_BYTES 2      /* a=batch b=classes c=members */
#define ADN_Q_DENSE_FWD_PATH 3            /* a=batch b=in c=out -> ADN_PATH_* that AUTO picks */
#define ADN_Q_SM_COUNT 4
#define ADN_Q_LAUNCH_COUNT 5              /* kernels launched by this library so far */
#define ADN_Q_DENSE_BWD_PATH 6            /* a=batch b=in c=out */
#define ADN_Q_DENSE_FWD_WORKSPACE_BYTES 7 /* a=batch b=in c=out (0 when the SIMT path is taken) */
#define ADN_Q_PLANES_BYTES 8              /* a=rows b=cols -> bytes of a split-plane tensor */
#define ADN_Q_DENSE_BWD_P_WORKSPACE_BYTES 9 /* a=batch b=in c=out */
#define ADN_Q_COLSUM_WORKSPACE_BYTES 10   /* a=rows b=cols */
#define ADN_Q_CONV_STEM_BWD_WORKSPACE_BYTES 11 /* a=batch b=channels c=filters */
#define ADN_Q_PLANE_FORMAT 12             /* current ADN_PLANES_* */
#define ADN_Q_TMA_MAP_CACHE_HITS 13       /* TMA descriptor cache statistics */
#define ADN_Q_TMA_MAP_CACHE_MISSES 14
#define ADN_Q_HEAD_PATH 15                /* a=dim b=members -> 0: adn_head_group, 1: adn_head_group_wide */
#define ADN_Q_HEAD_WIDE_WORKSPACE_BYTES 16 /* a=batch b=dim c=members (adn_head_group_wide) */
#define ADN_Q_METRICS_WORKSPACE_BYTES 17  /* a=rows b=max dim c=ops (adn_metrics_group) */

const char* adn_last_error(void);
/* One-time, idempotent host-side initialisation (kernel attributes, driver entry
 * points).  Must be called once outside any CUDA-graph capture; the Python
 * binding does so when the library is loaded on a machine with a GPU. */
int adn_init(void);
int adn_query(int key, int64_t a, int64_t b, int64_t c, int64_t* out_host);
int adn_set_dense_path(int path);
/* Process-wide format of every split-plane tensor the *_p entry points read and write (default ADN_PLANES_F16, or
 * the ADN_PLANES=tf32|f16 environment variable).  Plane buffers written under one format must not be read under
 * the other; ADN_Q_PLANES_BYTES follows the current format. */
int adn_set_plane_format(int fmt);
/* fp16 planes cannot hold a finite |value| >= 65520.  Every kernel that writes planes raises a sticky device flag
 * when it meets one; this call copies the flag to *flag_host (synchronising `stream`) and optionally clears it.
 * The caller is expected to re-run the affected work under ADN_PLANES_TF32 (core/search.py does, per iteration). */
int adn_plane_overflow(int* flag_host, int reset, void* stream);

/*
 * y[batch,out] = act(x[batch,in] @ w[in,out] + b[out])      (b may be NULL)
 * Replaces tf.layers.dense + tf.nn.relu of
 *   adanet/examples/simple_dnn.py:72-86 (_SimpleDNNBuilder.build_subnetwork),
 * and the forward-only replay of frozen members,
 *   adanet/core/estimator.py:1785-1882 / adanet/core/iteration.py:568-579.
 * workspace: adn_query(ADN_Q_DENSE_FWD_WORKSPACE_BYTES) bytes (hi/lo TF32 operand
 * planes of the tensor-core path); may be NULL/0 when that query returns 0.
 */
int adn_dense_fwd(const float* x, const float* w, const float* b, float* y,
                  int64_t batch, int64_t in, int64_t out, int act,
                  void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Backward of one dense layer given dz = dLoss/d(pre-activation) [batch,out]:
 *   dw[in,out] = x^T @ dz          db[out] = colsum(dz)
 *   dx[batch,in] = (dz @ w^T) * (x_relu_mask ? (x > 0) : 1)   (skipped if dx NULL)
 * With x_relu_mask=1, x is the ReLU output of the previous layer, so dx is that
 * layer's dz directly.  Replaces the gradient half of optimizer.minimize(loss,
 * var_list) at adanet/examples/simple_dnn.py:103-110 (var_list isolation:
 * adanet/core/ensemble_builder.py:754,783).
 * workspace: adn_query(ADN_Q_DENSE_BWD_WORKSPACE_BYTES) bytes, 16B aligned.
 */
int adn_dense_bwd(const float* x, const float* w, const float* dz,
                  float* dx, float* dw, float* db,
                  int64_t batch, int64_t in, int64_t out, int x_relu_mask,
                  void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Head loss on [batch,dim] logits: loss_out[0] = mean loss; dlogits (nullable)
 * = dLoss/dlogits.  labels: int64[batch] class ids (softmax), or float
 * [batch,dim] targets passed through labels_f (mse / sigmoid).
 * Replaces head.create_estimator_spec(...).loss on subnetwork logits,
 *   adanet/core/ensemble_builder.py:756-758 (+ :571-583).
 * workspace: adn_query(ADN_Q_HEAD_WORKSPACE_BYTES, batch, dim, 1).
 * = adn_head_loss_p(..., dlogits_planes = NULL, dlogits_colsum = NULL, dz_log2_scale = 0, ...).
 */
int adn_head_loss(int head, const float* logits, const int64_t* labels, const float* labels_f,
                  float* loss_out, float* dlogits, int64_t batch, int64_t dim,
                  void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Fused AdaNet ensemble head for one candidate ensemble of n_members:
 *   ens[b,c]  = bias[c] + sum_k w_k (.) member_k[b,c]         weighted.py:433-453,545-561
 *   loss      = head(ens, labels)                              ensemble_builder.py:416-420
 *   reg       = sum_k gamma_k * ||w_k||_1                      weighted.py:563-604
 *   adanet    = loss + reg                                     ensemble_builder.py:423-426
 *   dw_k      = d(loss + reg_multiplier*reg)/dw_k, dbias       weighted.py:606-617
 *               (reg_multiplier = 2 reproduces the reference's double-counted
 *                regulariser on the Ensembler.build_train_op path; 1 = legacy path)
 * members_host: host array of n_members device pointers to [batch,dim] logits.
 * w: device [n_members] (SCALAR) or [n_members,dim] (VECTOR).  MATRIX: members
 *    arrive pre-multiplied (last_layer_k @ W_k via adn_dense_fwd) and w is device
 *    float[n_members] holding ||W_k||_1 (adn_l1_norm); dw must be NULL and the
 *    caller forms dW_k = last_layer_k^T @ dens with adn_dense_bwd.
 * gammas_host: host array of lambda*r(h_k)+beta.  reg_is_zero: lambda==beta==0.
 * out3: device float[3] = {loss, reg, adanet_loss}.
 * dw (nullable): same shape as w.  dbias (nullable): [dim].
 * dens (nullable): [batch,dim] dLoss/d(ens) (needed for MATRIX weight grads).
 * ens_out (nullable): [batch,dim] ensemble logits (predict / evaluate).
 * A one-op adn_head_group: the adn_head_op of the same fields, colsum_only = 0, dz_log2_scale = 0, dens_planes =
 * NULL; errors as there, except dim > 64 is ADN_ERR_UNSUPPORTED.
 */
int adn_ensemble_head(int head, int mixture_type, const float* const* members_host, int n_members,
                      const float* w, const float* bias, const float* gammas_host, int reg_is_zero,
                      float reg_multiplier, const int64_t* labels, const float* labels_f,
                      float* out3, float* dw, float* dbias, float* dens, float* ens_out,
                      int64_t batch, int64_t dim, void* workspace, int64_t workspace_bytes, void* stream);

/*
 * TF1 optimizer update over n_tensors parameter tensors of one candidate.
 * params/grads/slot0/slot1: host arrays of device pointers; sizes_host: element
 * counts.  hyper_host: SGD {lr}; MOMENTUM {lr, momentum}; RMSPROP {lr, rho, mu,
 * eps}; ADAM {lr, beta1, beta2, eps}.  step_dev (nullable; required for ADAM):
 * device int64 count of updates already applied; the kernel uses *step_dev+1
 * for Adam's bias correction and the call increments it afterwards on the same
 * stream, so a captured CUDA graph replays correctly.  n_tensors <= 32.
 * Replaces optimizer.minimize's apply half at
 *   adanet/examples/simple_dnn.py:110 and adanet/ensemble/weighted.py:616.
 */
int adn_opt_step(int kind, float* const* params_host, const float* const* grads_host,
                 float* const* slot0_host, float* const* slot1_host, const int64_t* sizes_host,
                 int n_tensors, const float* hyper_host, int64_t* step_dev, void* stream);

/*
 * ---- plane-native dense pipeline (csrc/planes.cu, csrc/plane_fmt.cuh) ---------------
 * A *split-plane tensor* of a matrix T[rows, cols] is a pair of 11-significant-bit
 * planes, ADN_PLANES_F16: hi = fp16(T), lo' = fp16((T - hi) * 2^11), k-block = 64
 * columns; ADN_PLANES_TF32: hi = rna_tf32(T), lo = rna_tf32(T - hi), k-block = 32
 * columns; each stored k-block-major [ceil(cols/BK)][rows][BK] (zero padded in cols),
 * hi followed by lo followed by sign bits [ceil(cols/32)][rows] in one buffer of
 * adn_query(ADN_Q_PLANES_BYTES) bytes, 256 B aligned, ZERO-INITIALISED by the caller
 * once (the K padding must stay zero).  It is the operand format of the tensor-core GEMM
 * (3 MMAs per product: hi*hi, hi*lo, lo*hi): the same planes are read K-major or
 * MN-major by TMA, so forward, dX and dW all consume them without a transposed copy,
 * and each GEMM's epilogue writes the planes its consumer reads.
 * Gradient planes carry dz * 2^dz_log2_scale (fp16 has 5 exponent bits; the scale is
 * a power of two chosen by the caller, 0 for TF32 planes): dxp keeps the scale, every
 * fp32 output (dw, dx, dx_colsum) is returned un-scaled.
 * The per-layer calls below replace the same reference arithmetic as adn_dense_fwd /
 * adn_dense_bwd (adanet/examples/simple_dnn.py:72-86,103-110) for a whole subnetwork
 * whose activations never leave the plane format.
 */
int adn_planes_split(const float* src, int64_t rows, int64_t cols, void* planes, void* stream);
/* planes of src * 2^log2_scale (gradient tensors) */
int adn_planes_split_scaled(const float* src, int64_t rows, int64_t cols, void* planes, int log2_scale, void* stream);
int adn_planes_merge(const void* planes, int64_t rows, int64_t cols, float* dst, void* stream);
/* y = act(x @ w + b): xp planes [batch,in], wp planes [in,out]; result as planes (yp) or
 * dense fp32 row-major (y) -- exactly one of the two is non-NULL.  A one-op adn_dense_fwd_p_group: bias = b, no
 * dropout, n_srcs = 0. */
int adn_dense_fwd_p(const void* xp, const void* wp, const float* b, void* yp, float* y,
                    int64_t batch, int64_t in, int64_t out, int act, void* stream);
/* Backward of one dense layer from planes: dzp planes [batch,out] holding dz * 2^dz_log2_scale.
 *   dw[in,out] (dense, nullable) = x^T dz
 *   dx = (dz w^T) * (x_relu_mask ? x > 0 : 1) as planes (dxp) or dense (dx); both may be NULL
 *   dx_colsum[in] (nullable) = column sums of dx = the bias gradient of the layer below
 * workspace: adn_query(ADN_Q_DENSE_BWD_P_WORKSPACE_BYTES).  A one-op adn_dense_bwd_p_group: dx_mul = 1. */
int adn_dense_bwd_p(const void* xp, const void* wp, const void* dzp, void* dxp, float* dx,
                    float* dx_colsum, float* dw, int64_t batch, int64_t in, int64_t out,
                    int x_relu_mask, int dz_log2_scale, void* workspace, int64_t workspace_bytes, void* stream);
/*
 * Grouped forms: the same layer wave of several subnetworks (all candidates of an AdaNet iteration consume
 * the same minibatch, adanet/core/iteration.py:185-192) in ONE persistent launch per GEMM kind, so launch,
 * prologue and pipeline fill/drain are paid once per wave and narrow candidates hide behind wide ones.
 * Each op is checked before anything is launched; ops must not alias each other's outputs.  An output plane
 * buffer (yp, dxp) that is not aligned as the plane-tensor contract above asks is ADN_ERR_INVALID.
 */
/* One more input piece of a multi-source forward op: planes xp [batch, in] and the matching rows of the layer's
 * kernel as their own planes wp [in, out].  A dense layer over concat([x_0, x_1, ...], axis=-1) with kernel
 * W = [W_0; W_1; ...] (row blocks in the same order) is y = act(x_0 W_0 + x_1 W_1 + ... + b): AdaNet subnetworks
 * that read the hidden layers of earlier subnetworks (Cortes et al., ICML 2017; adanet/subnetwork/generator.py:96-105). */
typedef struct adn_fwd_src {
  const void* xp;
  const void* wp;
  int64_t in;          /* > 0 */
} adn_fwd_src;
#define ADN_FWD_MAX_SRCS 3 /* pieces per op besides (xp, wp) */
typedef struct adn_fwd_op {
  const void* xp;      /* planes [batch, in]  */
  const void* wp;      /* planes [in, out]    */
  const float* bias;   /* [out] or NULL       */
  void* yp;            /* planes [batch, out] -- exactly one of yp / y */
  float* y;            /* dense  [batch, out] */
  int64_t in, out;
  int32_t act;         /* ADN_ACT_* */
  int32_t reserved;
  /* tf.layers.dropout on the layer's output in TRAIN mode (adanet/examples/simple_dnn.py:80-81); planes out only.
   * dropout_rate 0 = none.  keep iff hash32(seed, layer, *dropout_step_dev, (dropout_row0 + row) * out + col) >=
   * rate * 2^32 (the mask is injected data shared with the oracle: oracle/adanet_oracle.py dropout_keep_mask), kept
   * values are multiplied by 1 / (1 - rate), and the sign bits (= the backward mask) follow the dropped-out values.
   * dropout_row0 (>= 0, 0 = a whole minibatch): the first minibatch row of this op's rows when the op runs a row slice
   * (a row-sharded candidate), so that every slice draws its rows of the whole minibatch's mask. */
  float dropout_rate;
  uint32_t dropout_seed;
  int32_t dropout_layer;
  int32_t dropout_row0;
  const int64_t* dropout_step_dev;
  /* Multi-source forward: y = act(xp wp + sum_{s < n_srcs} srcs[s].xp srcs[s].wp + b), K = in + sum_s srcs[s].in.
   * 0 <= n_srcs <= ADN_FWD_MAX_SRCS (srcs may be NULL when 0).  Ops with n_srcs > 0 run on a launch of their own,
   * so a group that mixes both kinds takes one launch per kind (per 8 ops); the epilogue (bias, ReLU, sign bits,
   * dropout, planes or dense out) is the same.  A negative or too large n_srcs, a NULL piece pointer, in <= 0 or
   * a misaligned plane buffer is ADN_ERR_INVALID before any op of the call is launched. */
  const adn_fwd_src* srcs;
  int32_t n_srcs;
  int32_t reserved3;
} adn_fwd_op;
typedef struct adn_bwd_op {
  const void* xp;      /* planes [batch, in]  */
  const void* wp;      /* planes [in, out]; required when dx is requested */
  const void* dzp;     /* planes [batch, out] of dz * 2^dz_log2_scale */
  void* dxp;           /* planes [batch, in] or NULL (same scale as dzp) */
  float* dx;           /* dense  [batch, in] or NULL (at most one of dxp / dx) */
  float* dx_colsum;    /* [in] or NULL */
  float* dw;           /* dense [in, out] or NULL */
  int64_t in, out;
  int32_t x_relu_mask;
  int32_t dz_log2_scale;
  void* workspace;     /* adn_query(ADN_Q_DENSE_BWD_P_WORKSPACE_BYTES, batch, in, out); one per op */
  int64_t workspace_bytes;
  float dx_mul;        /* dx is multiplied by this (0 = 1): 1 / (1 - rate) below a dropped-out activation x */
  float reserved2;
} adn_bwd_op;
int adn_dense_fwd_p_group(const adn_fwd_op* ops_host, int n, int64_t batch, void* stream);
int adn_dense_bwd_p_group(const adn_bwd_op* ops_host, int n, int64_t batch, void* stream);

/* adn_head_loss that also emits, in the same pass, dlogits * 2^dz_log2_scale as split planes (nullable) and the
 * (un-scaled) column sums of dlogits = the bias gradient of the logits layer (nullable): what the backward
 * GEMMs consume.  A one-op adn_head_group: head, members_host = &logits, n_members = 1, mixture_type = SCALAR,
 * reg_is_zero = 1, colsum_only = 1, labels, labels_f, dens = dlogits, dens_planes = dlogits_planes, dz_log2_scale,
 * dbias = dlogits_colsum, out3 = 16 bytes of the workspace past the op's own share, then loss_out[0] = out3[0].
 * workspace: adn_query(ADN_Q_HEAD_WORKSPACE_BYTES, batch, dim, 1).  Errors as adn_head_group, except dim > 64 is
 * ADN_ERR_UNSUPPORTED. */
int adn_head_loss_p(int head, const float* logits, const int64_t* labels, const float* labels_f,
                    float* loss_out, float* dlogits, void* dlogits_planes, float* dlogits_colsum,
                    int dz_log2_scale, int64_t batch, int64_t dim, void* workspace, int64_t workspace_bytes,
                    void* stream);
/* out[c] = sum_r x[r,c], fixed order (bias gradient of the logits layer).
 * workspace: adn_query(ADN_Q_COLSUM_WORKSPACE_BYTES). */
int adn_colsum(const float* x, int64_t rows, int64_t cols, float* out, void* workspace,
               int64_t workspace_bytes, void* stream);
/* adn_opt_step that also refreshes the split planes of 2-D parameters: planes_host[t]
 * (nullable per tensor) is the plane tensor of parameter t viewed as [size/cols, cols]. */
int adn_opt_step_p(int kind, float* const* params_host, const float* const* grads_host,
                   float* const* slot0_host, float* const* slot1_host, const int64_t* sizes_host,
                   int n_tensors, const float* hyper_host, int64_t* step_dev,
                   void* const* planes_host, const int64_t* cols_host, void* stream);

/*
 * Grouped heads: every subnetwork loss and every candidate-ensemble head of the candidates on one GPU in ONE launch
 * (plus one finalize launch) per 24 ops, over the same minibatch; above 512 CTAs (batch > 65536) op by op, three
 * launches each.  adn_ensemble_head and adn_head_loss(_p) are one-op calls of it.  All ops share batch (> 0) and
 * dim (1..64).  Every op is checked before anything is launched: a call that returns an error has written nothing.
 * An op is an ensemble head (colsum_only = 0) over n_members member logits:
 *   out3 = {loss, reg, loss + reg} of ens = bias + sum_k w_k (.) member_k (adn_ensemble_head), and on request
 *   dw = d(loss + reg_multiplier * reg)/dw, dbias, dens = dLoss/d(ens), ens_out = ens.
 * or a subnetwork loss (colsum_only = 1): members_host[0] = the logits (n_members = 1), out3[0] = mean loss,
 * dens / dens_planes = dlogits dense / as planes times 2^dz_log2_scale, dbias = column sums of dlogits = the
 * logits-layer bias gradient; w, bias, gammas and dw are ignored and reg = 0.
 */
typedef struct adn_head_op {
  int32_t head;              /* ADN_HEAD_* */
  int32_t mixture_type;      /* ADN_MIX_*; SCALAR for a subnetwork loss */
  const float* const* members_host; /* host array of n_members device pointers to [batch, dim] logits */
  int32_t n_members;         /* 1..64; members x dim must fit shared memory */
  int32_t reg_is_zero;       /* 1: lambda == beta == 0, no penalty */
  const float* w;            /* device: SCALAR [n_members], VECTOR [n_members, dim], MATRIX L1 norms [n_members];
                                NULL = all 1 */
  const float* bias;         /* device [dim] or NULL */
  const float* gammas_host;  /* host [n_members]: lambda * r(h_k) + beta; required unless reg_is_zero */
  float reg_multiplier;      /* weight of reg in dw (see adn_ensemble_head) */
  int32_t dz_log2_scale;     /* -60..60: dens_planes hold dLoss/d(ens) * 2^dz_log2_scale */
  const int64_t* labels;     /* device int64 [batch] class ids (softmax) */
  const float* labels_f;     /* device [batch, dim] targets (mse / sigmoid) */
  float* out3;               /* device float[3], required */
  float* dw;                 /* device, shape of w, or NULL; must be NULL for MATRIX */
  float* dbias;              /* device [dim] or NULL */
  float* dens;               /* device [batch, dim] dLoss/d(ens) or NULL */
  float* ens_out;            /* device [batch, dim] ensemble logits or NULL */
  void* dens_planes;         /* split planes [batch, dim] of dLoss/d(ens) * 2^dz_log2_scale or NULL */
  int32_t colsum_only;       /* 1: a subnetwork loss, see above */
  int32_t reserved;
  void* workspace;           /* device, required: adn_query(ADN_Q_HEAD_WORKSPACE_BYTES, batch, dim, n_members) */
  int64_t workspace_bytes;
} adn_head_op;
int adn_head_group(const adn_head_op* ops_host, int n, int64_t batch, int64_t dim, void* stream);
/* adn_head_group for heads of any width: the same ops, outputs and checks, on a kernel that keeps no shared-memory
 * copy of the members, so neither dim <= 64 nor the members x dim fit applies.  dim 1..16384 and n_members 1..64,
 * anything else is ADN_ERR_UNSUPPORTED; each op's workspace is adn_query(ADN_Q_HEAD_WIDE_WORKSPACE_BYTES, batch, dim,
 * n_members) instead.  adn_query(ADN_Q_HEAD_PATH, dim, n_members) says which of the two an op runs on.  Every
 * reduction runs in an order fixed by (batch, dim, n_members).  One head launch and one finalize launch per 24 ops. */
int adn_head_group_wide(const adn_head_op* ops_host, int n, int64_t batch, int64_t dim, void* stream);
/* Per-step bookkeeping of n candidate ensembles in one launch: state <- zero-debiased EMA of out3[2] (adn_ema_update)
 * and trace[(*step_dev % capacity)][0..3] = {*sub_loss, out3[0], out3[2], ema} (adn_record_scalars).  Every entry is
 * checked before anything is launched: a call that returns an error has written nothing. */
typedef struct adn_head_book {
  float* ema_state;
  const float* out3;
  const float* sub_loss;
  float* trace;
  float decay;
  int32_t capacity;
} adn_head_book;
int adn_head_bookkeeping(const adn_head_book* books_host, int n, const int64_t* step_dev, void* stream);

/* Grouped form of adn_opt_step_p: every optimizer of a training step (the subnetworks' and the mixture weights' of
 * every candidate on the GPU) in one launch.  Field meaning as the arguments of adn_opt_step_p.  Two ops of one call
 * must not share a step_dev.  Every op is checked before anything is launched: a call that returns an error has
 * changed no parameter, slot, plane or step counter. */
typedef struct adn_opt_op {
  int32_t kind;
  int32_t n_tensors;
  float* const* params_host;
  const float* const* grads_host;
  float* const* slot0_host;
  float* const* slot1_host;
  const int64_t* sizes_host;
  const float* hyper_host;
  int64_t* step_dev;
  void* const* planes_host;     /* nullable */
  const int64_t* cols_host;     /* nullable */
} adn_opt_op;
int adn_opt_step_group(const adn_opt_op* ops_host, int n, void* stream);

/*
 * Streaming evaluation metrics of the v2 BinaryClassHead and RegressionHead (AUC, precision, recall, means): the
 * accumulator half of the tf.keras metrics that the reference's Evaluator streams every hold-out batch through
 * (adanet/core/evaluator.py:97-140) and that Estimator.evaluate reports through the head's eval_metric_ops
 * (adanet/core/eval_metrics.py:111-118).
 * One op is one ensemble's fp32 logits [rows, dim] (the ens_out of its head) and its float labels [rows, dim]; the
 * call ADDS the batch to the op's accumulators (the caller zeroes them when an evaluation starts):
 *   sums[3] (fp64) += {sum of predictions, sum of labels, rows * dim}, where a prediction is the logit (MEANS) or
 *     p = 1.f / (1.f + expf(-logit)) in fp32 (BINARY);
 *   BINARY only, counts[ADN_METRICS_COUNTS] (int64) +=
 *     [0, 201): histogram of the negative examples over buckets b = #{i : t_i < p}, thresholds t_0 = fp32(-1e-7),
 *               t_i = fp32(i / 199) for i = 1..198, t_199 = fp32(1 + 1e-7) (Keras AUC(num_thresholds=200)); a NaN p
 *               is in bucket 0 (predicted negative at every threshold);
 *     [201, 402): the same histogram of the positive examples;
 *     [402], [403]: negatives, positives with logit > 0 (class_ids = argmax([0, logit]) of the v2 binary head).
 *   An example is positive when label > 0.5 (a NaN label is negative).  tp_i = sum_{b > i} positives[b] and so on
 *   are suffix sums of the histograms, formed on the host with the metric formulas (adanet_b200/core/metrics.py).
 * Counts are integer atomics; the sums go through per-CTA partials in `workspace` and one fixed-order finalize, and
 * the CTA count is a function of (rows, max dim, n) alone, so results are bit-identical across runs and devices.
 * One launch plus one finalize launch per 32 ops.  Every op is checked before anything is launched: n outside
 * 1..ADN_METRICS_MAX_OPS, rows or dim < 1, a null pointer (counts may be NULL for MEANS), a bad kind or two ops
 * sharing `sums` is ADN_ERR_INVALID, BINARY with dim != 1 ADN_ERR_UNSUPPORTED, a workspace smaller than
 * adn_query(ADN_Q_METRICS_WORKSPACE_BYTES, rows, max dim, n) ADN_ERR_WORKSPACE; a rejected call changes no
 * accumulator.
 */
#define ADN_METRICS_BINARY 0      /* dim == 1, sigmoid head: histograms, class-id counts and sums */
#define ADN_METRICS_MEANS 1       /* regression head: sums only */
#define ADN_METRICS_THRESHOLDS 200
#define ADN_METRICS_COUNTS 404    /* 2 * (ADN_METRICS_THRESHOLDS + 1) + 2 */
#define ADN_METRICS_MAX_OPS 1024
typedef struct adn_metrics_op {
  int32_t kind;             /* ADN_METRICS_* */
  int32_t reserved;
  const float* logits;      /* device [rows, dim] */
  const float* labels_f;    /* device [rows, dim] */
  int64_t dim;
  int64_t* counts;          /* device [ADN_METRICS_COUNTS], accumulated; NULL for MEANS */
  double* sums;             /* device [3], accumulated */
} adn_metrics_op;
int adn_metrics_group(const adn_metrics_op* ops_host, int n, int64_t rows, void* workspace, int64_t workspace_bytes,
                      void* stream);

/* out[0] = sum_i |x[i]| over n elements (tf.norm(ord=1), weighted.py:573), fixed order. */
int adn_l1_norm(const float* x, int64_t n, float* out, void* stream);

/* dw[i] += coef * sign(w[i]): the complexity-regulariser term of a MATRIX mixture weight's gradient,
 * coef = reg_multiplier * gamma_k (adanet/ensemble/weighted.py:563-617; SCALAR / VECTOR weights get it
 * inside adn_ensemble_head). */
int adn_l1_grad_add(float* dw, const float* w, int64_t n, float coef, void* stream);

/*
 * SimpleCNN stem (adanet/examples/tutorials/customizing_adanet.ipynb, SimpleCNNBuilder.build_subnetwork):
 *   Conv2D(filters, kernel_size=3, padding="same", activation="relu") -> MaxPool2D(2, 2) -> Flatten   [Keras, NHWC]
 * images [batch, height, width, channels] fp32, kernel [3, 3, channels, filters] (HWIO), bias [filters].
 * Forward writes the flattened pooled features [batch, (height/2)*(width/2)*filters] (h, w, c order) as a
 * split-plane tensor (adn_query(ADN_Q_PLANES_BYTES, batch, cols), zero-initialised) -- the input format of
 * adn_dense_fwd_p, sign bits = ReLU/pool mask -- plus a 2-bit argmax per element (16 per word,
 * [batch, cols/16] uint32) that routes the gradient like TF's MaxPoolGrad (first maximum in scan order).
 * Backward takes the gradient w.r.t. the pooled features as dense fp32 [batch, cols] already multiplied by
 * (pooled > 0) -- adn_dense_bwd_p(..., dx=dense, x_relu_mask=1) of the first dense layer produces exactly
 * that -- and returns dkernel [3,3,channels,filters] and dbias [filters] (fixed-order reduction).  No gradient
 * w.r.t. the images is formed (the stem is the first layer).
 * height, width even; channels in {1, 3}; filters in {16, 32, 48, 64}; (height + 2) * (width + 2) * channels
 * <= 24576.  Every shape the forward accepts, the backward accepts too.
 * workspace: adn_query(ADN_Q_CONV_STEM_BWD_WORKSPACE_BYTES, batch, channels, filters).
 */
int adn_conv_stem_fwd(const float* images, const float* kernel, const float* bias, void* out_planes,
                      uint32_t* argmax, int64_t batch, int height, int width, int channels, int filters,
                      void* stream);
int adn_conv_stem_bwd(const float* images, const uint32_t* argmax, const float* dpooled, float* dkernel,
                      float* dbias, int64_t batch, int height, int width, int channels, int filters,
                      void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Zero-debiased EMA of the AdaNet loss (adanet/core/candidate.py:117-129 ->
 * assign_moving_average(zero_debias=True)).  state: device float[3] =
 * {biased, n, value}; loss: device float*.
 */
int adn_ema_update(float* state, const float* loss, float decay, void* stream);

/*
 * Step bookkeeping that must live on the device so a whole training step can be
 * captured in a CUDA graph (replaces the per-spec `step` variables and hooks of
 * adanet/core/iteration.py:150-205,961-996):
 *   adn_record_scalars: trace[(*step_dev % capacity)*stride + i] = *src_host[i], i < n (n <= 16)
 *   adn_counter_add:    *counter_dev += delta
 */
int adn_record_scalars(const float* const* src_host, int n, float* trace, int64_t stride,
                       const int64_t* step_dev, int64_t capacity, void* stream);
int adn_counter_add(int64_t* counter_dev, int64_t delta, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ADANET_B200_H_ */
