/*
 * adaptive_b200.h -- C ABI of libadaptive_b200.so (hand-written sm_90a CUDA).
 *
 * Drop-in boundary for the predict()/add_examples() hot path of codelion/adaptive-classifier.
 * The reference has no FFI of its own: the seams are Python object calls into third-party
 * libraries (SURVEY.md section 8(b)).  Every entry point below names the reference call site it
 * replaces (paths relative to /root/reference/).  The ctypes binding a maintainer would add is in
 * INTEGRATION.md; adaptive_classifier_b200/_cabi.py is that binding.
 *
 * Conventions
 *   - plain C types only; `ac_stream_t` is a cudaStream_t passed as void* (NULL = default stream).
 *   - unless a name ends in `_host`, every data pointer is a DEVICE pointer owned by the caller.
 *   - all matrices are row-major, fp32, ids int64 unless stated; no hidden allocation after
 *     `*_create` / explicit workspaces.
 *   - return value: 0 = ok, negative = error (AC_E_*); text via ac_last_error() (thread-local).
 *   - no CPU fallback exists: with no usable sm_90 (H100) device every compute call returns AC_E_CUDA.
 */
#ifndef ADAPTIVE_B200_H
#define ADAPTIVE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void *ac_stream_t;

enum {
    AC_OK = 0,
    AC_E_INVALID = -1,   /* bad argument (shape, null pointer, k > limit ...) */
    AC_E_CUDA = -2,      /* CUDA runtime / launch failure, or no sm_90 device */
    AC_E_WORKSPACE = -3, /* workspace too small */
    AC_E_UNSUPPORTED = -4
};

int ac_version(void);                 /* ABI version, currently 1 */
const char *ac_last_error(void);      /* thread-local message of the last failing call */
int ac_device_check(void);            /* 0 when the current device is sm_90 (H100), else AC_E_CUDA */


/* ------------------------------------------------------------------------------------------
 * Stage K -- prototype kNN.  Replaces faiss.IndexFlatL2.search at
 *   src/adaptive_classifier/memory.py:110-114 (call sites :34,106,113,114,158,159,164,172,182,190)
 * ------------------------------------------------------------------------------------------ */

/* algo selector for ac_knn_l2_topk */
enum {
    AC_KNN_AUTO = 0,
    AC_KNN_EXACT = 1,   /* fp32 SIMT exact scan + radix select (any k <= AC_KNN_MAX_K)       */
    AC_KNN_TENSOR = 2   /* wgmma coarse pass (.f16 over the fp16 shadow, or .tf32) + exact fp32 re-rank,
                           k <= AC_KNN_TENSOR_MAX_K.  k <= 16: per-query certification against the rigorous coarse
                           error bound; uncertified queries -- and every query when k > 16 -- take a second,
                           device-conditional tensor pass that collects the provable superset {d~ <= tau + 2 eps},
                           re-ranked exactly (indices identical to AC_KNN_EXACT either way; no host sync) */
};
#define AC_KNN_MAX_K 2048
#define AC_KNN_TENSOR_MAX_K 1024

/* bytes of scratch ac_knn_l2_topk needs for these sizes (device memory, 256-byte aligned) */
int ac_knn_workspace_bytes(int B, int64_t N, int D, int k, int algo, size_t *bytes);

/*
 * out_d[B,k] ascending squared-L2 distances, out_i[B,k] int64 row ids (+row_offset); ties -> lower id;
 * when N < k the tail is (+inf, -1)  [IndexFlatL2.search semantics, memory.py:113-114,121].
 * Distances are the exact fp32 lane-ordered sum restated in oracle/knn_oracle.c (bit-identical).
 * p_sqnorm[N] (nullable) = cached ||p||^2 for the tensor path; computed into the workspace if NULL.
 * p_half (nullable) = fp16 shadow copy of P[N,D] (ac_knn_make_shadow): the tensor path then runs its coarse pass as
 *   wgmma .f16 over 2.N.D bytes (D %% 64 == 0); candidates are still re-ranked on the fp32 rows, so the
 *   result is the same bits either way.
 * stats (nullable, device int32[4], ACCUMULATED): [0] queries that needed the second tensor pass, [1] queries whose
 *   2-eps band overflowed the candidate buffer (their rows of out_d/out_i are NOT exact: the caller must redo them with
 *   AC_KNN_EXACT), [2] max rows collected for one query, [3] searches.  With stats != NULL the call never synchronises
 *   (graph-capturable); with stats == NULL it synchronises once at the end and recomputes overflowed queries itself.
 */
int ac_knn_l2_topk(const float *Q, const float *P, const float *p_sqnorm, const void *p_half,
                   int B, int64_t N, int D, int k,
                   float *out_d, int64_t *out_i, int64_t row_offset,
                   void *workspace, size_t workspace_bytes, int algo, int32_t *stats, ac_stream_t stream);

/* fp16 (RNE) shadow of the prototype matrix for the tensor path's coarse pass; out_half holds N*D halves */
int ac_knn_make_shadow(const float *P, int64_t N, int D, void *out_half, ac_stream_t stream);

/* ||p||^2 per row (fp32), the cache the tensor path consumes */
int ac_row_sqnorm(const float *P, int64_t N, int D, float *out, ac_stream_t stream);

/* multi-shard merge (new: row-sharded index over G GPUs, SURVEY.md section 8(e)); d[G,B,k], i[G,B,k]
 * -> k smallest by (d, i); entries with i < 0 ignored.  Bit-identical to a single-shard search. */
int ac_topk_merge(const float *d, const int64_t *i, int G, int B, int k,
                  float *out_d, int64_t *out_i, ac_stream_t stream);

/* memory.py:117,128-134: scores[b,:] = softmax_k(exp(-d[b,:])); entries with idx < 0 get 0 */
int ac_proto_scores(const float *d, const int64_t *idx, int B, int k, float *scores, ac_stream_t stream);

/* memory.py:149-150 (prototype = mean of the class's retained examples): rows X[n,D] with class id
 * cls[n] in [0,C) -> mean[C,D], count[C]; classes with no rows keep mean = 0 */
int ac_segment_mean(const float *X, const int32_t *cls, int64_t n, int D, int C,
                    float *mean, int32_t *count, ac_stream_t stream);

/* Device-resident maintenance of the per-class example store for a whole add_examples() call (SURVEY.md 8(f) N2).
 * Replaces the per-example sequence memory.py:60-72 (append, prune when over max_examples_per_class) / :196-217
 * (_prune_examples: keep the `cap` embeddings nearest the mean of the cap + 1, list reordered by that distance) /
 * :138-153 (_update_prototype = mean of the retained embeddings).
 *   rows  [n_slots, cap + 1, D]  class stores;  order [n_slots, cap + 1]: a permutation of the physical slots 0..cap per class,
 *   positions [0, count) = the stored rows in list order, positions [count, cap] = free slots;  count [n_slots].
 *   new_rows [*, D]; new_index [n_new]: row numbers of new_rows grouped by touched class, arrival order inside a class;
 *   cls_start [n_touched + 1]: offsets of the groups in new_index;  touched [n_touched]: class slot of every group.
 * One CTA per touched class processes its new examples sequentially (example j sees the list example j - 1 left).
 * Outputs: src_out [n_touched, cap]: provenance of every retained list position (< old count: that position of the old list,
 * >= old count: old count + index of the new example inside its group, -1: empty); proto_out [n_touched, D].
 * workspace: n_touched * D * 8 bytes. */
int ac_memory_append_prune(float *rows, int32_t *order, int32_t *count, int cap, int D, const float *new_rows,
                           const int32_t *new_index, const int32_t *cls_start, const int32_t *touched, int n_touched,
                           int32_t *src_out, float *proto_out, void *workspace, size_t workspace_bytes, ac_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Stage H -- adaptive head.  Replaces nn.Module.__call__ / autograd / AdamW on AdaptiveHead:
 *   forward  src/adaptive_classifier/models.py:71-80, classifier.py:428-442, :1341-1354
 *   training classifier.py:333-351, :1489-1505, multilabel.py:387-397
 * Weights in nn.Linear layout: W0[H0,D], W1[H1,H0], W2[C,H1]  (H0 = D, H1 = D/2 in the reference).
 * ------------------------------------------------------------------------------------------ */
enum { AC_ACT_LOGITS = 0, AC_ACT_SOFTMAX = 1, AC_ACT_SIGMOID = 2 };
enum { AC_LOSS_CE = 0, AC_LOSS_BCE = 1, AC_LOSS_CE_STRATEGIC = 2 };

typedef struct {
    int D, H0, H1, C;
    float *W0, *b0, *W1, *b1, *W2, *b2;
} ac_head_params;

/* eval-mode forward (dropout inactive).  out[B,C]; scratch >= B*(H0+H1) floats */
int ac_head_forward(const float *X, int B, const ac_head_params *p, int act,
                    float *out, float *scratch, size_t scratch_floats, ac_stream_t stream);

typedef struct {
    float lr, beta1, beta2, eps, weight_decay, max_norm; /* AdamW + clip_grad_norm_ */
    int step;                /* 1-based count of this update (bias correction) */
    int loss_kind;           /* AC_LOSS_CE: targets int64[B]; AC_LOSS_BCE: targets float[B,C] */
    float dropout_p;         /* 0.1 in the reference; 0 disables */
    const float *mask0;      /* optional injected dropout masks [B,H0], [B,H1] holding 0 or 1/(1-p);   */
    const float *mask1;      /*   NULL -> Philox masks from (seed, step)                                */
    uint64_t seed;
    /* optional EWC term (ewc.py:96-115): grad += 2*lambda/B * F*(theta-theta*) over the first
       ewc_rows_out rows of the output layer (the head may have grown), NULL = off */
    const ac_head_params *ewc_fisher;
    const ac_head_params *ewc_star;
    float ewc_lambda;
    int ewc_C_old;
    /* AC_LOSS_CE_STRATEGIC only (0 otherwise): the batch is [x_1..x_n ; br_1..br_n] with n = n_regular, and the step minimises
       mean CE(x) + strategic_lambda / n * sum over the best-response rows whose first-argmax differs from y of CE(br) */
    int n_regular;
    float strategic_lambda;
} ac_train_cfg;

/* bytes of workspace for a training / gradient call with `batch` rows per step and n_steps steps (1 for a single step) */
int ac_head_train_workspace_bytes(int batch, int n_steps, const ac_head_params *p, size_t *bytes);

/* one optimizer step: fwd(train) + loss + bwd + [EWC grad] + global-norm clip + AdamW, as one launch of the persistent
 * cooperative kernel of csrc/head_train.cuh (B <= 64; D, H0, H1 multiples of 4).
 * m, v: AdamW moments (same shapes as p).  out_stats[0] = task loss, [1] = ewc penalty,
 * [2] = grad norm before clipping (device floats). */
int ac_head_train_step(const float *X, const void *targets, int B,
                       ac_head_params *p, ac_head_params *m, ac_head_params *v,
                       const ac_train_cfg *cfg, float *out_stats,
                       void *workspace, size_t workspace_bytes, ac_stream_t stream);

/* one EPOCH of the reference's training loops (classifier.py:329-353, :1485-1507; multilabel.py:381-399) in one call:
 * X[n,D], targets (int64[n] or float[n,C]) and the shuffled index list perm[n] (what the reference's DataLoader with
 * torch.Generator().manual_seed(42) yields) live on the device; batches of `batch` rows (last one partial) are gathered
 * and stepped inside ONE kernel launch (the grid stays resident for the whole epoch: parameters live in shared memory, six
 * grid barriers per step).  cfg->step = 1-based number of the first update.  loss_accum (nullable): [0] += task loss + EWC
 * penalty per step.  step_stats (nullable): [ceil(n / batch), 3] = (task loss, EWC penalty, grad norm before clipping) of
 * every step -- what the reference's loop reads back with loss.item() (classifier.py:353, :1507).
 * workspace: ac_head_train_workspace_bytes(batch, ceil(n / batch), ...). */
int ac_head_train_epoch(const float *X, const void *targets, const int64_t *perm, int n, int batch,
                        ac_head_params *p, ac_head_params *m, ac_head_params *v, const ac_train_cfg *cfg,
                        float *loss_accum, float *step_stats, void *workspace, size_t workspace_bytes, ac_stream_t stream);

/* diagnostic: per-phase time of the training kernel: nanoseconds three observed CTAs (one per layer of the head) spent in each
 * of the 7 phases and 6 grid barriers of a step (13 counters) and inside the product routines (7 counters from index 14), summed
 * over all steps since enabled.  enable != 0 starts accumulating; out72_host (nullable) receives 3 x 24 counters. */
int ac_head_phase_timing(int enable, unsigned long long *out72_host);
/* diagnostic: launch plan of the training kernel: out5 = {CTAs, operand-ring stages, AdamW moments resident in shared memory (0/1),
 * dynamic shared-memory bytes, reserved} */
int ac_head_train_plan(int batch, const ac_head_params *p, int *out5);

/* gradient only (no update) of mean CE/BCE wrt all parameters, eval mode: the building block of
 * EWC._compute_fisher (ewc.py:67-92).  fisher += grad^2 * inv_n_batches when fisher != NULL */
int ac_head_grad(const float *X, const void *targets, int B, const ac_head_params *p, int loss_kind,
                 ac_head_params *grad_out, ac_head_params *fisher_accum, float inv_n_batches,
                 float *out_loss, void *workspace, size_t workspace_bytes, ac_stream_t stream);

/* ewc.py:105-115: out[0] = lambda/bs * sum F*(theta-theta*)^2 over the parameters (C_old rows of the
 * output layer) */
int ac_ewc_penalty(const ac_head_params *p, const ac_head_params *fisher, const ac_head_params *star,
                   float lambda, float inv_batch, int C_old, float *out, ac_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Stage S -- strategic mode.  Replaces the per-sample Python loops of
 *   strategic.py:74-123   SeparableCostFunction.compute_best_response / _generate_candidates (50 head forwards per sample)
 *   strategic.py:200-242  StrategicOptimizer.strategic_loss
 *   classifier.py:1602-1647 AdaptiveClassifier._strategic_training_step
 * The candidate set of a row x (D >= 5) is fixed: candidate 0 is x, candidate 1 + 10 i + j (i = 0..3, j = 0..9) and
 * 41 + j (i = 4, j = 0..8) is x with x_i replaced by fl(x_i + delta[j]), delta = torch.linspace(-2, 2, 10).  The utility of a
 * candidate y is max softmax(head(y)) - cost(x, y); the first maximum wins (NaN never does; no winner -> candidate 0).
 *   AC_COST_LINEAR     relu(c1 . (y - x)) = relu(fl(c1_i * fl(y_i - x_i)))       (LinearCostFunction, bit-exact)
 *   AC_COST_SEPARABLE  relu(c2 . y - c1 . x), both dots in one fixed order       (SeparableCostFunction)
 * ------------------------------------------------------------------------------------------ */
enum { AC_COST_LINEAR = 0, AC_COST_SEPARABLE = 1 };
#define AC_STRATEGIC_CANDIDATES 50

typedef struct {
    int cost_kind;           /* AC_COST_* */
    const float *c1;         /* [D] device: alpha (linear) or c1 (separable) */
    const float *c2;         /* [D] device: c2 (separable; ignored for linear) */
    float delta[10];         /* torch.linspace(-2, 2, 10) in fp32, built on the host */
    float dropout_p;         /* train-mode candidate forwards (0 = eval mode) */
    uint64_t seed;           /* dropout key: (seed, step, row, candidate), a stream apart from the training kernel's masks */
    int step;
} ac_strategic_cfg;

/* bytes of workspace for ac_strategic_best_response on B rows */
int ac_strategic_workspace_bytes(int B, const ac_head_params *p, size_t *bytes);

/* best response of every row of X[B,D] against the head p: out_choice[B] (candidate index 0..49), out_utility[B] (its utility),
 * out_Y[B,D] (nullable: the chosen candidate, bit for bit).  D >= 5; D, H0, H1 multiples of 4. */
int ac_strategic_best_response(const float *X, int B, const ac_head_params *p, const ac_strategic_cfg *cfg, int32_t *out_choice,
                               float *out_utility, float *out_Y, void *workspace, size_t workspace_bytes, ac_stream_t stream);

/* bytes of workspace for ac_head_train_strategic on n stored rows */
int ac_head_train_strategic_workspace_bytes(int n, const ac_head_params *p, size_t *bytes);

/* the whole _strategic_training_step on the device with no host synchronisation: for each of n_epochs epochs, batches of
 * min(16, n) rows of X[n,D] / targets int64[n] are taken in the order perms[epoch * n ..] (what the reference's DataLoader with
 * torch.Generator().manual_seed(42) yields), their best responses are searched in train mode (scfg->dropout_p, seed, step),
 * and one AdamW step runs on the 2B rows [x ; br] with AC_LOSS_CE_STRATEGIC (cfg->strategic_lambda; cfg->step = first step,
 * cfg->loss_kind and cfg->n_regular are ignored).  step_stats[n_steps, 3] (device) = (strategic loss, 0, grad norm before
 * clipping) of every step. */
int ac_head_train_strategic(const float *X, const int64_t *targets, const int64_t *perms, int n, int n_epochs, ac_head_params *p,
                            ac_head_params *m, ac_head_params *v, const ac_train_cfg *cfg, const ac_strategic_cfg *scfg,
                            float *step_stats, void *workspace, size_t workspace_bytes, ac_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Stage E -- encoder.  Replaces `self.model(**inputs).last_hidden_state[:,0,:]` + F.normalize at
 *   src/adaptive_classifier/classifier.py:1271-1275 (HF BertModel / RobertaModel / ModernBertModel / NomicBertModel /
 *   JinaEmbeddingsV3Model / EuroBertModel forward).
 * ------------------------------------------------------------------------------------------ */
enum { AC_ARCH_BERT = 0, AC_ARCH_ROBERTA = 1, AC_ARCH_MODERNBERT = 2,
       AC_ARCH_MPNET = 3 /* post-LN BERT block, RoBERTa positions, relative position bias (rel_bias); head_dim 64 */,
       AC_ARCH_DEBERTA = 4 /* DeBERTa-v2/v3: post-LN BERT block, BERT positions, disentangled c2p + p2c attention
                              (pos_key, pos_query, pos_span, rel_index); head_dim 64 */,
       AC_ARCH_ROTARY = 5 /* NomicBERT, jina-embeddings-v3: post-LN BERT block, RoPE on q and k (rope_full, positions
                             0..S-1 for every sequence, padded or not), embeddings LayerNorm(word + type) with no position
                             table (pos_emb is not read); head_dim 64, no embedding projection */,
       AC_ARCH_EUROBERT = 6 /* EuroBERT: ModernBERT's pre-norm block with RMSNorm (ln_eps = rms_norm_eps), no embedding norm
                               (the residual stream starts as the raw embed_tokens rows), RoPE on q and k (rope_full, positions
                               0..S-1 for every sequence, padded or not), full attention in every layer, no biases,
                               ffn_act = AC_FFN_SWIGLU; head_dim 64, no embedding projection.  Weights: see ac_encoder_weights */ };
#define AC_ENCODER_MAX_S 512   /* longest sequence ac_encoder_forward_cls accepts for BERT / RoBERTa / DistilBERT (their
                                  position tables stop at 512).  An AC_ARCH_ROBERTA encoder whose table has more than
                                  AC_ENCODER_MAX_S + pad_idx + 1 rows (XLM-R: bge-m3, arctic-embed-l-v2.0, 8194 rows) accepts
                                  S <= min(AC_MODERNBERT_MAX_S, max_pos - pad_idx - 1) */
#define AC_MODERNBERT_MAX_S 8192   /* largest max_pos of an AC_ARCH_MODERNBERT encoder (max_position_embeddings of the
                                      published checkpoints) */
enum {
    AC_PREC_TF32 = 0,   /* wgmma .tf32 on fp32 storage (kNN coarse pass, ac_linear_tc tests) */
    AC_PREC_F16 = 1     /* wgmma .f16 with fp16 operands (RNE from fp32; same 10-bit mantissa as tf32),
                           fp32 accumulation; the encoder's precision: 1.7e-4 on distances, bf16 would be 1.4e-3 */
};

typedef struct {
    int arch;            /* AC_ARCH_* */
    int layers, hidden, heads, intermediate;   /* hidden % 128 == 0; head_dim = hidden / heads is 64 or 32
                                                  (64 only for AC_ARCH_MODERNBERT, AC_ARCH_MPNET, AC_ARCH_DEBERTA,
                                                  AC_ARCH_ROTARY and AC_ARCH_EUROBERT) */
    int vocab, max_pos, type_vocab;
    int pad_idx;         /* roberta, mpnet: position ids start at pad_idx+1 */
    float ln_eps;
    int precision;       /* AC_PREC_* */
    int max_tokens;      /* workspace is sized for B*S <= max_tokens */
    int cls_only;        /* != 0: the last layer's output projection / FFN / LayerNorms run on the CLS rows only
                            (classifier.py:1272 uses nothing else); 0 keeps the full last hidden state */
    /* AC_ARCH_MODERNBERT only (ignored otherwise), except rope_full, which AC_ARCH_ROTARY and AC_ARCH_EUROBERT read too.
       For all three,
       AC_ENCODER_MAX_S <= max_pos <= AC_MODERNBERT_MAX_S is the longest sequence the encoder accepts and the rows of its
       RoPE tables (RoPE has no position parameters). */
    int sliding_window;          /* half-window w = local_attention / 2: a sliding layer's query i sees keys |i - j| <= w */
    const int32_t *layer_sliding;  /* HOST array [layers]: 1 = sliding_attention, 0 = full_attention (config.layer_types) */
    const float *rope_full;      /* DEVICE [max_pos, 64] fp32 RoPE table of the full-attention layers (every layer of
                                    AC_ARCH_ROTARY and AC_ARCH_EUROBERT):                                              */
    const float *rope_sliding;   /*   row = position, [0, 32) cos, [32, 64) sin of the 32 frequencies (HF
                                       ModernBertRotaryEmbedding's formula = LlamaRotaryEmbedding's, default rope type,
                                       built by the caller); the sliding layers' table */
    /* AC_ARCH_MPNET only (ignored otherwise), copied by ac_encoder_create.  DEVICE [heads, 2 AC_ENCODER_MAX_S - 1] fp32:
       entry (h, AC_ENCODER_MAX_S - 1 + key - query) is the bias every layer adds to head h's scaled score of (query, key)
       (HF MPNetEncoder.compute_position_bias: relative_attention_bias.weight[bucket(key - query), h], built by the caller) */
    const float *rel_bias;
    /* AC_ARCH_DEBERTA only (ignored otherwise), read by ac_encoder_create, which gathers them into fp16 (RNE) attention
       operands; all DEVICE.  For query i and key j, r = i - j, every layer l adds to the unscaled score q_i . k_j
           q_i . pos_key[l, c(r), head]  +  k_j . pos_query[l, c(r), head]
       and scales the sum by 1 / sqrt(3 head_dim) (HF DisentangledSelfAttention with pos_att_type c2p|p2c). */
    const float *pos_key;        /* [layers, 2 pos_span, H] fp32: key_proj(rel) (share_att_key) or pos_key_proj(rel), with
                                    rel = rel_embeddings (LayerNorm-ed when norm_rel_ebd = layer_norm), biases included */
    const float *pos_query;      /* [layers, 2 pos_span, H] fp32: query_proj(rel) or pos_query_proj(rel) */
    int pos_span;                /* position_buckets, or max_relative_positions without buckets */
    const int32_t *rel_index;    /* [2 R - 1] int32, R = rel_radius or AC_ENCODER_MAX_S when it is 0: entry R - 1 + r is
                                    c(r) = clamp(bucket(r) + pos_span, 0, 2 pos_span - 1) (HF build_relative_position)
                                    for -R < r < R */
    /* factorized embeddings (ALBERT, ELECTRA): width E of the embedding tables and their LayerNorm; 0 means hidden.  An E
       other than hidden needs the projection ac_encoder_weights.emb_proj_w; with a projection E % 128 == 0, E <= hidden. */
    int embedding_size;
    int ffn_act;                 /* AC_FFN_*: the FFN activation of a post-LN encoder; AC_ARCH_MODERNBERT (GeGLU) takes 0,
                                    AC_ARCH_EUROBERT AC_FFN_SWIGLU; among the others AC_FFN_SWIGLU is AC_ARCH_ROTARY's only */
    int rel_radius;              /* AC_ARCH_DEBERTA: the radius R of rel_index.  0 = AC_ENCODER_MAX_S, with S <= max_pos.
                                    AC_ENCODER_MAX_S < R <= AC_MODERNBERT_MAX_S: S <= R, for an encoder without absolute
                                    positions only (position_biased_input = False: pos_emb all zeros, which
                                    ac_encoder_create checks).  Must be 0 for every other arch.  The handle keeps
                                    layers x (2 D + 1) x heads x 64 KiB of relative operands, D <= 5 for the published
                                    settings (D = the block offset past which c(r) is saturated, derived from rel_index). */
} ac_encoder_config;

enum {
    AC_FFN_GELU_ERF = 0,         /* exact-erf GELU (HF "gelu") */
    AC_FFN_GELU_TANH = 1,        /* tanh-approximated GELU (HF "gelu_new", "gelu_pytorch_tanh"; ALBERT v2) */
    AC_FFN_SWIGLU = 2            /* down(silu(gate_proj x) * up_proj x) (NomicBERT): ff1_w[l] is [2I, H], the activated rows
                                    (gate_proj) then the multiplier rows (up_proj); ff1_b[l] is [2I] */
};

/* device pointers to the HF state_dict tensors (fp32, HF layout [out,in]).
 * AC_ARCH_MODERNBERT (models/modernbert/modeling_modernbert.py, every bias absent) uses only
 *   word_emb   embeddings.tok_embeddings      emb_ln_w  embeddings.norm
 *   ao_w       layers.l.attn.Wo               ao_ln_w   layers.l.mlp_norm
 *   ff2_w      layers.l.mlp.Wo
 * and the fields after out_ln_b; every other pointer may be NULL.
 * AC_ARCH_ROTARY takes the BERT fields but pos_emb, every bias present (pass zeros where the checkpoint has none): q/k/v/ao
 * self_attn.{q,k,v,o}_proj, ao_ln post_attention_layernorm, ff1 mlp.fc1 or (AC_FFN_SWIGLU) cat(mlp.gate_proj, mlp.up_proj),
 * ff2 mlp.fc2 / mlp.down_proj, out_ln post_mlp_layernorm.
 * AC_ARCH_EUROBERT (models/eurobert/modeling_eurobert.py, no biases) uses the AC_ARCH_MODERNBERT fields, every other pointer
 * may be NULL (emb_ln_w is not read: there is no embedding norm):
 *   word_emb        embed_tokens                      attn_norm_w[l]  layers.l.input_layernorm (entry 0 USED)
 *   wqkv[l]         cat(q_proj, k_proj, v_proj) [3H, H], k_proj / v_proj expanded to every query head (grouped-query
 *                   attention: query head h reads kv head h / (heads / num_key_value_heads), HF repeat_kv's order)
 *   ao_w[l]         layers.l.self_attn.o_proj         ao_ln_w[l]      layers.l.post_attention_layernorm
 *   wi[l]           cat(mlp.gate_proj, mlp.up_proj) [2I, H]
 *   ff2_w[l]        layers.l.mlp.down_proj            final_norm_w    norm
 * Shared layers (ALBERT's cross-layer parameter sharing): a packed operand whose source pointers -- weights, biases and the
 * LayerNorm folded into it -- equal an earlier layer's reuses that layer's packed copy, so pass the same pointer for every
 * layer that shares a tensor.  Sharing is by pointer identity only: equal values at different addresses are packed twice. */
typedef struct {
    /* width embedding_size when it is set (ALBERT, ELECTRA), else hidden */
    const float *word_emb, *pos_emb, *type_emb, *emb_ln_w, *emb_ln_b;
    /* arrays of `layers` device pointers each (host arrays of device pointers) */
    const float *const *q_w, *const *q_b, *const *k_w, *const *k_b, *const *v_w, *const *v_b;
    const float *const *ao_w, *const *ao_b, *const *ao_ln_w, *const *ao_ln_b;
    const float *const *ff1_w, *const *ff1_b, *const *ff2_w, *const *ff2_b;
    const float *const *out_ln_w, *const *out_ln_b;
    /* AC_ARCH_MODERNBERT (and AC_ARCH_EUROBERT, as listed above) */
    const float *const *attn_norm_w;  /* [layers] layers.l.attn_norm (ModernBERT: entry 0 unused, layer 0's attn_norm is
                                         Identity) */
    const float *final_norm_w;        /* final_norm */
    const float *const *wqkv;         /* [layers] layers.l.attn.Wqkv [3H, H], q, k, v thirds */
    const float *const *wi;           /* [layers] layers.l.mlp.Wi [2I, H], input rows then gate rows */
    /* embedding projection E -> H after the embedding LayerNorm: ALBERT encoder.embedding_hidden_mapping_in, ELECTRA
       embeddings_project.  NULL = none (the embeddings are the residual stream).  AC_ARCH_BERT / AC_ARCH_ROBERTA only:
       the projection runs AFTER the embedding LayerNorm (ALBERT / ELECTRA order; DeBERTa-v2's embed_proj, which runs
       before it, is not implemented). */
    const float *emb_proj_w;          /* [H, E] */
    const float *emb_proj_b;          /* [H] */
} ac_encoder_weights;

typedef struct ac_encoder ac_encoder;

/* copies + repacks the weights (fused QKV, operand rounding) and allocates the activation workspace */
int ac_encoder_create(const ac_encoder_config *cfg, const ac_encoder_weights *w, ac_encoder **out);
int ac_encoder_destroy(ac_encoder *enc);

/* ids[B,S] int32 token ids, mask[B,S] int32 (1 keep / 0 pad; NULL = all ones), type_ids nullable (ignored by
 * AC_ARCH_MODERNBERT, whose RoPE positions are 0..S-1 for every sequence, padded or not).  S <= AC_ENCODER_MAX_S, or
 * S <= max_pos for AC_ARCH_MODERNBERT, AC_ARCH_ROTARY and AC_ARCH_EUROBERT, or, for an AC_ARCH_ROBERTA encoder with max_pos > AC_ENCODER_MAX_S + pad_idx + 1,
 * S <= min(AC_MODERNBERT_MAX_S, max_pos - pad_idx - 1) (its positions run from pad_idx + 1; head_dim 64 past
 * AC_ENCODER_MAX_S), or, for an AC_ARCH_DEBERTA encoder created with rel_radius > AC_ENCODER_MAX_S, S <= rel_radius.
 * out_unit_cls[B,H] = L2-normalised (eps 1e-12) CLS row of the last hidden state. */
int ac_encoder_forward_cls(ac_encoder *enc, const int32_t *ids, const int32_t *mask,
                           const int32_t *type_ids, int B, int S, float *out_unit_cls,
                           ac_stream_t stream);


/* debugging / parity: copy the full last hidden state [B*S,H] of the previous forward */
int ac_encoder_last_hidden(ac_encoder *enc, float *out, int64_t n_floats, ac_stream_t stream);

/* debugging / parity: run this encoder's attention stage alone.  qk [B*S, 2H] fp16 (q then k, head h at columns h*dh),
 * vT fp16 in the layout the QKV epilogue writes ((b*H + feature) * S_pad + key, S_pad = roundup(S, 8); the pad keys may
 * hold any finite value), mask as in ac_encoder_forward_cls, window = sliding half-window (keys |query - key| <= window;
 * 0 = full; must be 0 unless AC_ARCH_MODERNBERT), cls_rows != 0 computes the first 128-query block only (later rows of
 * ctx_out are then unspecified).  ctx_out [B*S, H] fp16 = softmax(q k^T / sqrt(dh) + rel_bias + mask) v per head; a query
 * with no valid key in reach gets zeros.  Uses the encoder's heads, head_dim and rel_bias, and accepts and refuses the
 * shapes ac_encoder_forward_cls does.  On an AC_ARCH_DEBERTA encoder the scores are those of layer 0: (q k^T + c2p + p2c)
 * / sqrt(3 dh) with layer 0's pos_key / pos_query.  All pointers DEVICE. */
int ac_encoder_attention(ac_encoder *enc, const void *qk, const void *vT, const int32_t *mask, int B, int S, int window,
                         int cls_rows, void *ctx_out, ac_stream_t stream);

/* debugging / parity: run one projection of layer `layer` alone on caller-supplied inputs, with this encoder's packed
 * operands, buffers and fused epilogue, exactly as ac_encoder_forward_cls runs it.  M = B*S <= max_tokens rows; fp16
 * arrays are row-major, stats / stats_out are [M] (mu, r) float pairs (RMSNorm: (0, r)).
 *   AC_PROJ_EMB        a = LayerNorm-ed embedding rows [M, E] fp16 -> out0 y = a Wp^T + bp [M, H] fp32, out1 fp16(y)
 *                      (encoders with an embedding projection only)
 *   AC_PROJ_QKV        a = fp16 residual sums [M, H], stats of the norm the layer's QKV consumes ((0, 1) where that is
 *                      the identity) -> out0 q | k [M, 2H] fp16 (RoPE with the layer's table on rotary encoders), out1 V^T
 *                      [B*H, S_pad] fp16 at (b*H + feature) * S_pad + key, S_pad = roundup(S, 8); pad keys unspecified
 *   AC_PROJ_WO, _W2    a = attention context [M, H] / FFN activations [M, I] fp16, y = residual sums [M, H] fp32 and
 *                      their stats -> out0 y_new = a W^T + b + LN_pending(y) [M, H] fp32, out1 fp16(y_new), stats_out the
 *                      statistics of y_new.  LN_pending is what the forward leaves pending there: post-LN, the previous
 *                      layer's output LayerNorm before Wo (the identity in layer 0) and the attention-output LayerNorm
 *                      before W2; pre-LN, the identity (stats are then not read)
 *   AC_PROJ_FFN1       a = fp16 residual sums [M, H], stats of the norm FFN1 consumes -> out0 activations [M, I] fp16
 *   AC_PROJ_FFN1_ROWS  the CLS-only tail's FFN1 (cls_only encoders, last layer): a = normalised rows [M, H] fp16 -> out0
 *                      activations [M, I] fp16
 * Unused pointers may be NULL.  Overwrites the handle's activation buffers.  All pointers DEVICE. */
enum { AC_PROJ_EMB = 0, AC_PROJ_QKV = 1, AC_PROJ_WO = 2, AC_PROJ_FFN1 = 3, AC_PROJ_W2 = 4, AC_PROJ_FFN1_ROWS = 5 };
int ac_encoder_projection(ac_encoder *enc, int layer, int role, int B, int S, const void *a, const float *y,
                          const float *stats, void *out0, void *out1, float *stats_out, ac_stream_t stream);

/* generic tensor-core linear (the encoder's GEMM with its fused epilogues), exposed for parity tests and roofline
 * measurement: Y[M,N] = epi(X[M,K] W[N,K]^T + bias) (+ residual).  epi: 0 bias, 1 bias+GELU(erf), 2 bias+fp32 residual,
 * 3 bias+GELU(tanh) (AC_PREC_F16 with out_half != 0 only), 4 SwiGLU (AC_PREC_F16 with out_half != 0, N % 64 == 0): W's
 * rows interleaved in 32-row groups (rows 64 g .. + 31 activated, 64 g + 32 .. + 63 their multipliers), Y [M, N / 2] with
 * Y[m, 32 g + j] = silu(p[m, 64 g + j]) * p[m, 64 g + 32 + j], p = X W^T + bias.
 * precision AC_PREC_TF32: X, W, Y fp32 (operands used as stored; round_out != 0 rounds Y to tf32);
 * precision AC_PREC_F16 : X, W fp16, Y fp32 or (out_half != 0, epi != 2) fp16. */
int ac_linear_tc(const void *X, const void *W, const float *bias, const float *residual, void *Y,
                 int M, int N, int K, int epi, int round_out, int precision, int out_half, ac_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Stage T -- tokenization.  Replaces `self.tokenizer(texts, max_length=..., truncation=True, padding=True)` at
 *   src/adaptive_classifier/classifier.py:1259-1265 for WordPiece tokenizers of the BERT shape: BertNormalizer,
 *   BertPreTokenizer, WordPiece, post-processor "[special] A [special]", right truncation and padding, added tokens with
 *   normalized = false and single_word = false.  Which tokenizers qualify, and the tables below, are decided and built by
 *   adaptive_classifier_b200/tokenizer.py from the installed `tokenizers` library.
 * ------------------------------------------------------------------------------------------ */
#define AC_TOKENIZER_CODEPOINTS 0x110000

typedef struct {
    /* HOST tables over every codepoint c < AC_TOKENIZER_CODEPOINTS:
       norm[c]: bit 31 set = c normalizes to itself; else bits 5..29 = offset into pool and bits 0..4 = length of its normalized
                expansion (bit 30 on an empty expansion: canonical ordering does not cross it);
       cls[c]:  bits 0-1 the pre-tokenizer class of c as a normalized char (0 other, 1 whitespace, 2 punctuation), bits 2-7 its
                rank in canonical ordering (0 for starters; marks of lower rank move before marks of higher rank) */
    const uint32_t *norm;
    const uint8_t *cls;
    const uint32_t *pool;
    int64_t pool_len;
    /* vocab entry v: the bytes vocab_bytes[vocab_offsets[v] .. vocab_offsets[v + 1]) with id vocab_ids[v] */
    const uint8_t *vocab_bytes;
    const int64_t *vocab_offsets;
    const int32_t *vocab_ids;
    int n_vocab;
    /* added tokens matched on the raw text (leftmost, then longest), same layout */
    const uint8_t *added_bytes;
    const int64_t *added_offsets;
    const int32_t *added_ids;
    int n_added;
    const char *prefix;          /* continuing_subword_prefix, <= 16 bytes, not NUL-terminated */
    int prefix_len;
    int cls_id, sep_id, pad_id, unk_id;   /* first and last special token of the template, padding, WordPiece unk_token */
    int max_input_chars;         /* WordPiece max_input_chars_per_word: longer words (in chars) are unk_id */
} ac_tokenizer_spec;

typedef struct ac_tokenizer ac_tokenizer;
/* copies the tables and builds the vocab's hash table on the device */
int ac_tokenizer_create(const ac_tokenizer_spec *spec, ac_tokenizer **out);
int ac_tokenizer_destroy(ac_tokenizer *tok);
/* bytes of workspace ac_tokenize needs for B texts */
int ac_tokenize_workspace_bytes(const ac_tokenizer *tok, int B, size_t *bytes);
/* text: UTF-8 bytes of B >= 1 texts, text i = text[offsets[i] .. offsets[i + 1]) (offsets int64[B + 1], nondecreasing, within
 * the buffer).  Ids equal the library's for valid UTF-8; an invalid byte is read as U+FFFD, and no text is read past its end.
 * tokens[B, max_length]: row i starts with the lengths[i] ids of text i, [CLS] pieces [SEP] truncated to max_length >= 2; *max_len = max lengths[i].
 * Every pointer is DEVICE; nothing synchronises. */
int ac_tokenize(const ac_tokenizer *tok, const uint8_t *text, const int64_t *offsets, int B, int max_length, int32_t *tokens,
                int32_t *lengths, int32_t *max_len, void *workspace, size_t workspace_bytes, ac_stream_t stream);
/* ids / mask / type_ids (nullable) [B, S], S <= max_length (the batch's longest, read back by the caller): the first lengths[i]
 * tokens of row i, then the pad id with mask 0; type ids 0.  DEVICE pointers. */
int ac_tokenize_pack(const ac_tokenizer *tok, const int32_t *tokens, const int32_t *lengths, int B, int max_length, int S,
                     int32_t *ids, int32_t *mask, int32_t *type_ids, ac_stream_t stream);

/* Byte-level BPE tokenizers (RoBERTa, ModernBERT, EuroBERT): no normalizer, the pre-tokenizer ByteLevel(use_regex) with the
 * GPT-2 split or Split(Llama-3 pattern) + ByteLevel, a BPE model without dropout, affixes or byte fallback whose vocab holds
 * all 256 byte symbols, "[special] A [special]", right truncation and padding, added tokens with single_word = false.  The
 * same handle type and calls as above, with two differences:
 *   - ac_tokenize_workspace_bytes refuses a BPE handle: its workspace depends on the batch's text bytes, so ask
 *     ac_tokenize_workspace_bytes_text (which answers for either kind);
 *   - ac_tokenize on a BPE handle takes max_len int32[2]: max_len[0] = max lengths[i] over the texts it tokenized, and
 *     max_len[1] = 1 when it left texts to the caller (0 otherwise), each with lengths[i] = -1.  Those are the texts among whose
 *     first max_length - 2 words is one longer than AC_BPE_MAX_WORD bytes (or that do not fit the workspace); the caller
 *     tokenizes them on the host and writes their rows and lengths before ac_tokenize_pack. */
#define AC_BPE_MAX_WORD 1024
#define AC_BPE_SPLIT_GPT2 0     /* 's|'t|'re|'ve|'m|'ll|'d| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+ */
#define AC_BPE_SPLIT_LLAMA3 1   /* (?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+ */

typedef struct {
    /* HOST class byte of every codepoint c < AC_TOKENIZER_CODEPOINTS, as the library's regex engine and Rust see it: bit 0
       \p{L}, bit 1 \p{N}, bit 2 \s, bit 3 Rust char::is_whitespace (lstrip / rstrip); bits 4-7 the letter c matches
       case-insensitively among s t r e v m l d (1 .. 8, 0 none; read by the Llama-3 contractions only) */
    const uint8_t *cls;
    int split;                   /* AC_BPE_SPLIT_GPT2 or AC_BPE_SPLIT_LLAMA3 */
    int add_prefix_space;        /* ByteLevel: a space in front of every piece that does not start with one (GPT-2 split only) */
    int ignore_merges;           /* a word that is a whole vocab entry is that entry */
    /* the model vocab as raw bytes (byte symbols mapped back), entry v = vocab_bytes[vocab_offsets[v] .. vocab_offsets[v + 1])
       with id vocab_ids[v]; read only with ignore_merges (may be NULL otherwise) */
    const uint8_t *vocab_bytes;
    const int64_t *vocab_offsets;
    const int32_t *vocab_ids;
    int n_vocab;
    const int32_t *byte_ids;     /* [256] the id of each byte's symbol */
    const int32_t *merges;       /* [n_merges, 3] left id, right id, merged id; the rank is the row */
    int n_merges;
    /* added tokens: bytes, offsets, ids as in ac_tokenizer_spec, and flags bit 0 normalized (matched after the others,
       inside the gaps they leave), bit 1 lstrip, bit 2 rstrip */
    const uint8_t *added_bytes;
    const int64_t *added_offsets;
    const int32_t *added_ids;
    const uint8_t *added_flags;
    int n_added;
    int cls_id, sep_id, pad_id;
} ac_bpe_tokenizer_spec;

int ac_tokenizer_create_bpe(const ac_bpe_tokenizer_spec *spec, ac_tokenizer **out);
/* bytes of workspace ac_tokenize needs for B texts of text_bytes bytes in all (offsets[B] - offsets[0]) at max_length */
int ac_tokenize_workspace_bytes_text(const ac_tokenizer *tok, int B, int64_t text_bytes, int max_length, size_t *bytes);

/* SentencePiece Unigram tokenizers of the XLM-RoBERTa shape (xlm-roberta-*, bge-m3, multilingual-e5-*, jina-embeddings-v3,
 * snowflake-arctic-embed-l-v2.0) as AutoTokenizer loads them: the normalizer Precompiled(charsmap) or none, the pre-tokenizer
 * Sequence[WhitespaceSplit, Metaspace("▁", prepend_scheme always, split)], a Unigram model without byte fallback,
 * "[special] A [special]", right truncation and padding, added tokens with single_word = false.  The same handle type and
 * calls as BPE: ac_tokenize_workspace_bytes refuses the handle, ac_tokenize takes max_len int32[2] and leaves to the caller
 * (lengths[i] = -1, max_len[1] = 1) the texts among whose first max_length - 2 words is one longer than AC_UNIGRAM_MAX_WORD
 * bytes ("▁" included) or whose normalized words do not fit the workspace. */
#define AC_UNIGRAM_MAX_WORD 4096

typedef struct {
    /* HOST class byte of every codepoint c < AC_TOKENIZER_CODEPOINTS: bit 0 c joins the grapheme cluster before it (Extend,
       ZWJ, SpacingMark), bit 1 a control (Control, CR, LF), bit 2 Prepend, bit 3 Rust char::is_whitespace */
    const uint8_t *cls;
    /* the Precompiled charsmap as (key, value) pairs, key k = map_keys[map_key_offsets[k] .. map_key_offsets[k + 1]) and its
       value likewise; n_map = 0 for a tokenizer without a normalizer */
    const uint8_t *map_keys;
    const int64_t *map_key_offsets;
    const uint8_t *map_values;
    const int64_t *map_value_offsets;
    int n_map;
    int grow;                    /* no value is longer than grow bytes per key byte (1 .. 64; 1 without a normalizer) */
    /* the model vocab in id order: piece v = piece_bytes[piece_offsets[v] .. piece_offsets[v + 1]) with score piece_scores[v] */
    const uint8_t *piece_bytes;
    const int64_t *piece_offsets;
    const double *piece_scores;
    int n_pieces;
    int unk_id;
    /* added tokens as in ac_bpe_tokenizer_spec */
    const uint8_t *added_bytes;
    const int64_t *added_offsets;
    const int32_t *added_ids;
    const uint8_t *added_flags;
    int n_added;
    int cls_id, sep_id, pad_id;
} ac_unigram_tokenizer_spec;

int ac_tokenizer_create_unigram(const ac_unigram_tokenizer_spec *spec, ac_tokenizer **out);

/* ------------------------------------------------------------------------------------------
 * predict_batch() glue on the device (classifier.py:1329-1384) and the end-to-end pipeline.
 * ------------------------------------------------------------------------------------------ */

/* memory.py:117-134 generalised to many rows per class (SURVEY.md section 8(d)): the k nearest rows (d asc, idx)
 * are mapped through row_class[global row id] (NULL: class = row id), a class keeps its nearest row,
 * out_score = softmax(exp(-d)) over the distinct classes; tails padded with (-1, 0).  k <= 32. */
int ac_proto_class_scores(const float *d, const int64_t *idx, const int32_t *row_class, int B, int k,
                          int32_t *out_cls, float *out_score, ac_stream_t stream);

/* the same for k up to 1024 (predict(): k = num_classes, classifier.py:424-425); class ids < n_classes <= 4096 */
int ac_proto_class_scores_n(const float *d, const int64_t *idx, const int32_t *row_class, int B, int k, int n_classes,
                            int32_t *out_cls, float *out_score, ac_stream_t stream);

/* predict() blend over ALL classes (classifier.py:446-480): combined[c] = proto_score[c] * w_proto[c] + head_probs[b,c] *
 * w_head[c] (per-class weights from training_history: < 10 examples -> 0.3 / 0.7, else 0.7 / 0.3), normalised by the sum,
 * top kout.  proto_cls / proto_score [B, kp] as written by ac_proto_class_scores(_n); head_probs [B, C] nullable. */
int ac_blend_dense(const int32_t *proto_cls, const float *proto_score, int kp, const float *head_probs, int B, int C,
                   const float *w_proto, const float *w_head, int kout, int32_t *out_cls, float *out_score, ac_stream_t stream);

/* classifier.py:1347-1350 (torch.topk of the head probabilities): out_neg_vals[B,k] holds the k largest values
 * NEGATED (ascending), out_idx[B,k] their column ids; ties -> lower id. */
int ac_topk_desc_workspace_bytes(int B, int C, int k, size_t *bytes);
int ac_topk_desc(const float *values, int B, int C, int k, float *out_neg_vals, int64_t *out_idx,
                 void *workspace, size_t workspace_bytes, ac_stream_t stream);

/* classifier.py:1358-1384: combined[label] = w_proto*proto + w_head*head, stable descending sort,
 * normalised by the sum, top k.  head_neg_val as produced by ac_topk_desc.  k, kh <= 32. */
int ac_blend_topk(const int32_t *proto_cls, const float *proto_score, const int64_t *head_idx,
                  const float *head_neg_val, int B, int k, int kh, float w_proto, float w_head,
                  int32_t *out_cls, float *out_score, ac_stream_t stream);

/* E -> K -> class scores -> H -> top-k -> blend with all intermediate buffers owned by the handle.
 * head may be NULL (prototype-only prediction).  row_class nullable. */
typedef struct ac_pipeline ac_pipeline;
int ac_pipeline_create(ac_encoder *enc, const float *P, const float *p_sqnorm, const void *p_half,
                       const int32_t *row_class, int64_t N, int D, const ac_head_params *head, int max_B, int S, int k,
                       int64_t row_offset, int shards /* 1, or the number of GPUs the rows are sharded over */, ac_pipeline **out);
int ac_pipeline_destroy(ac_pipeline *pl);
/* device buffers at the boundary (bench.py `value`) */
int ac_pipeline_predict_device(ac_pipeline *pl, const int32_t *ids_dev, const int32_t *mask_dev, int B,
                               int32_t *out_cls_dev, float *out_score_dev, ac_stream_t stream);
/* HOST buffers at the boundary (bench.py `e2e`): H2D of ids and D2H of the [B,k] result inside the call.  The device part of the
 * step is replayed as a CUDA graph from the third call with a batch size on (first: ordinary launches, second: capture) -- at B = 1
 * the ~110 launches of a step cost more host time than GPU time.  Results are identical to the
 * eager step; AC_PIPELINE_GRAPH=0 in the environment, or enabled per-kernel profiling (ac_profile_enable), keeps the step eager. */
int ac_pipeline_predict_host(ac_pipeline *pl, const int32_t *ids_host, int B, int32_t *out_cls_host,
                             float *out_score_host, ac_stream_t stream);
/* The phases of one step, for the row-sharded multi-GPU search (SURVEY.md section 8(e)): the caller (parallel.py) runs the
 * two collectives between them on the same stream -- all-gather of the unit embeddings, ONE all-to-all of the packed
 * (distance, id) candidates -- so that N > 1 executes the same kernels, with the same side-stream overlap of the head, as N = 1.
 *   ac_pipeline_encode         ids -> unit CLS rows (ac_pipeline_embeddings returns the device pointer, [B, D])
 *   ac_pipeline_search_shard   q_all[G*B, D] (rank-major) over THIS shard -> packed: G chunks of (d[B,k] fp32 | id[B,k] int64)
 *   ac_pipeline_finish_sharded received chunks (chunk g = shard g's candidates of MY queries) -> merge by (d, global id)
 *                              [bit-identical to the unsharded search] -> class scores -> head -> blend */
int ac_pipeline_encode(ac_pipeline *pl, const int32_t *ids_dev, const int32_t *mask_dev, int B, ac_stream_t stream);
int ac_pipeline_embeddings(ac_pipeline *pl, const float **emb_dev);
int ac_pipeline_search_shard(ac_pipeline *pl, const float *q_all, int G, int B, void *packed, ac_stream_t stream);
int ac_pipeline_finish_sharded(ac_pipeline *pl, const void *received, int G, int B, int32_t *out_cls_dev, float *out_score_dev,
                               ac_stream_t stream);
/* search statistics accumulated since the last reset (synchronises): see ac_knn_l2_topk `stats` */
int ac_pipeline_knn_stats(ac_pipeline *pl, int32_t *out4_host, int reset, ac_stream_t stream);
/* parity tests: copy the last call's unit CLS rows [B,D] and kNN result [B,k] into caller device buffers */
int ac_pipeline_debug_copy(ac_pipeline *pl, int B, float *emb_out, float *knn_d_out, int64_t *knn_i_out,
                           ac_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Measurement hooks (bench.py): number of kernels launched by this library so far, and optional
 * CUDA-event timing of the dominant kernels on their launching stream.
 * classes: 0 encoder wgmma GEMM, 1 attention, 2 kNN tensor pass 1, 3 kNN exact scan, 4 kNN tensor pass 2 (device-conditional)
 * ------------------------------------------------------------------------------------------ */
long long ac_launch_count(void);
int ac_profile_enable(int on);
int ac_profile_read(int cls, double *ms, double *flops, double *bytes, long long *launches);

#ifdef __cplusplus
}
#endif
#endif /* ADAPTIVE_B200_H */
