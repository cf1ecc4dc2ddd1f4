/* rpx.h — C ABI of the H100-native premise-retrieval engine (librpx.so).
 *
 * The reference (lean-dojo/ReProver) has NO plugin / operator / FFI interface for
 * this path: its seam is the Python attribute surface of `PremiseRetriever`
 * (retrieval/model.py:29) and `Corpus.get_nearest_premises` (common.py:299).  Each
 * entry point below therefore cites the reference Python call it replaces; the
 * Python shim `reprover_b200.retriever.B200PremiseRetriever` re-creates the
 * reference surface on top of these calls (see INTEGRATION.md).
 *
 * Conventions
 *   - extern "C", plain pointers / integers, no torch types, no C++ exceptions.
 *   - Every function returning `int` returns RPX_OK (0) or an RPX_ERR_* code; the
 *     message is available from rpx_last_error() (thread-local).
 *   - `d_` parameters are DEVICE pointers, `h_` parameters are HOST pointers.  The
 *     caller owns every buffer; the library borrows them for the duration of the
 *     stream-ordered work it enqueues and never frees them.  The only memory the
 *     library uses beyond its arguments is the explicit workspace / packed-weight
 *     buffers whose sizes it reports.
 *   - `stream` is a cudaStream_t passed as void*.  All work is enqueued on it;
 *     functions return without synchronising unless stated.
 *   - Handles are not thread-safe per handle; distinct handles are independent.
 *   - sm_90a (H100) only.  There is no CPU or other-GPU fallback: calling a
 *     compute entry point without such a device fails with RPX_ERR_CUDA /
 *     RPX_ERR_UNSUPPORTED.
 */
#ifndef RPX_H_
#define RPX_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RPX_VERSION 200 /* 0.2.0 */

enum {
  RPX_OK = 0,
  RPX_ERR_INVALID = 1,     /* bad argument */
  RPX_ERR_CUDA = 2,        /* a CUDA runtime / driver call failed */
  RPX_ERR_UNSUPPORTED = 3, /* valid request outside what the engine implements */
  RPX_ERR_WORKSPACE = 4,   /* workspace / packed buffer too small */
  RPX_ERR_MASK = 5         /* attention_mask is not a right-padded prefix mask */
};

enum { RPX_DTYPE_BF16 = 0, RPX_DTYPE_F32 = 1 };

/* Last error message of the calling thread ("" if none). */
const char* rpx_last_error(void);
int rpx_version(void);
/* RPX_OK iff the current CUDA device is compute capability 9.0. */
int rpx_device_check(void);

/* ------------------------------------------------------------------------- encoder
 * Replaces the HF `T5EncoderModel` forward that `PremiseRetriever._encode`
 * (retrieval/model.py:92-114) calls at :101-105, plus the masked mean-pool and
 * F.normalize at :108-114.  Architecture constants come from the checkpoint's
 * config.json (HF T5Config; ByT5-small values in SURVEY.md §8).
 */
typedef struct {
  int32_t vocab_size;       /* 384  */
  int32_t d_model;          /* 1472 */
  int32_t d_kv;             /* 64   */
  int32_t d_ff;             /* 3584 */
  int32_t num_layers;       /* 12   */
  int32_t num_heads;        /* 6    */
  int32_t rel_buckets;      /* 32   */
  int32_t rel_max_distance; /* 128  */
  float ln_eps;             /* 1e-6 */
} rpx_t5_config;

/* Raw HF weights, fp32, row-major, DEVICE pointers.  The per-layer members are
 * HOST arrays of `num_layers` device pointers.  Safetensors key for each member
 * is given on the right (i = layer). */
typedef struct {
  const float* d_shared;         /* shared.weight                                   [vocab, d_model]   */
  const float* d_rel_bias;       /* encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight [buckets, heads] */
  const float* d_final_ln;       /* encoder.final_layer_norm.weight                 [d_model]          */
  const float* const* h_q;       /* encoder.block.i.layer.0.SelfAttention.q.weight  [heads*d_kv, d_model] */
  const float* const* h_k;       /* ...k.weight                                                         */
  const float* const* h_v;       /* ...v.weight                                                         */
  const float* const* h_o;       /* ...o.weight                                     [d_model, heads*d_kv] */
  const float* const* h_ln0;     /* encoder.block.i.layer.0.layer_norm.weight       [d_model]          */
  const float* const* h_wi0;     /* encoder.block.i.layer.1.DenseReluDense.wi_0.weight [d_ff, d_model]  */
  const float* const* h_wi1;     /* ...wi_1.weight                                                      */
  const float* const* h_wo;      /* ...wo.weight                                    [d_model, d_ff]    */
  const float* const* h_ln1;     /* encoder.block.i.layer.1.layer_norm.weight       [d_model]          */
} rpx_t5_weights;

typedef struct rpx_encoder rpx_encoder; /* opaque */

/* Bytes of device memory the packed (bf16, RMSNorm-folded, FFN-interleaved)
 * weight image needs; the caller allocates it and keeps it alive while the
 * handle lives. */
size_t rpx_encoder_packed_bytes(const rpx_t5_config* cfg);

/* Builds the packed weight image on `stream` and returns a handle.
 * Mirrors `PremiseRetriever.load_hf` (retrieval/model.py:52-66) for the encoder
 * part: fp32 checkpoint -> bf16 compute copy. */
int rpx_encoder_create(const rpx_t5_config* cfg, const rpx_t5_weights* w, void* d_packed,
                       size_t packed_bytes, void* stream, rpx_encoder** out);
int rpx_encoder_destroy(rpx_encoder* enc);

/* Workspace needed to encode up to `max_tokens` packed tokens in `max_seqs`
 * sequences in one call. */
size_t rpx_encoder_workspace_bytes(const rpx_encoder* enc, int64_t max_tokens, int64_t max_seqs);

/* Tokenise + encode + pool + normalise `n_seqs` byte strings.
 * Replaces, per batch, the tokenizer call at retrieval/model.py:199-205 (ByT5:
 * id = byte + 3, EOS = 1 appended, truncation to max_seq_len INCLUDING the EOS;
 * HF tokenization_byt5.py:195-208) followed by `_encode` (:92-114).
 *   d_bytes     concatenated UTF-8 bytes of all sequences (device)
 *   h_offsets   n_seqs + 1 byte offsets into d_bytes (HOST; the host needs the
 *               lengths to size the launch)
 *   d_out       [n_seqs, d_model] unit-norm rows, RPX_DTYPE_BF16 or RPX_DTYPE_F32
 * If h_offsets is page-locked memory it must stay valid until `stream` reaches this call.
 * Strings must not contain ByT5 special-token literals ("</s>", "<pad>", "<unk>",
 * "<extra_id_N>"); callers route those through rpx_encode_ids (the Python shim does). */
int rpx_encode_bytes(rpx_encoder* enc, const uint8_t* d_bytes, const int64_t* h_offsets,
                     int32_t n_seqs, int32_t max_seq_len, void* d_out, int32_t out_dtype,
                     void* d_workspace, size_t workspace_bytes, void* stream);

/* Exact `_encode(input_ids, attention_mask)` signature (retrieval/model.py:92-94):
 * int64 [B, L] ids and mask on the device.  The mask must be a right-padded
 * prefix mask with at least one token per row (what the reference tokenizer call
 * produces); anything else returns RPX_ERR_MASK.  Synchronises `stream` once
 * (row lengths are read back to size the launch). */
int rpx_encode_ids(rpx_encoder* enc, const int64_t* d_input_ids, const int64_t* d_attention_mask,
                   int32_t batch, int32_t seq_len, void* d_out, int32_t out_dtype,
                   void* d_workspace, size_t workspace_bytes, void* stream);

/* The encoder's per-token output, `last_hidden_state` of HF `T5EncoderModel` (the final RMSNorm of every
 * token, modeling_t5.py:782), for callers that pool it themselves.  Replaces
 *   self.encoder(input_ids=..., attention_mask=..., return_dict=True).last_hidden_state   retrieval/model.py:101-105
 *   self.encoder(input_ids, attention_mask)[0]                                            retrieval/model.py:97-99
 * and the README's `model(tokenized_s.input_ids).last_hidden_state` (no mask).
 *   d_attention_mask  int64 [batch, seq_len], or NULL: HF's attention_mask=None, every position is a token
 *                     (pad id 0 included) and every row is seq_len long
 *   d_out             [batch, seq_len, d_model], RPX_DTYPE_BF16 or RPX_DTYPE_F32, 16-byte aligned; row (b, p)
 *                     is token p of sequence b.  Nothing past batch * seq_len rows is written.
 * Validation, workspace rule (rpx_encoder_workspace_bytes(enc, batch * seq_len, batch)), the id-range check
 * and the synchronisation are those of rpx_encode_ids; a non-NULL mask must be a right-padded prefix mask
 * (RPX_ERR_MASK otherwise).  Without a mask the length readback is skipped, but the call still synchronises
 * once to check the ids.  The one deliberate difference from HF: positions past a row's mask length are
 * written as zeros, where HF computes values for them (the pad queries attend to the real keys).  No code of the
 * reference reads them: `_encode` and the README both multiply the hidden states by the mask before pooling. */
int rpx_encode_ids_hidden(rpx_encoder* enc, const int64_t* d_input_ids,
                          const int64_t* d_attention_mask /* NULL: every position is a token */,
                          int32_t batch, int32_t seq_len, void* d_out /* [batch, seq_len, d_model] */,
                          int32_t out_dtype, void* d_workspace, size_t workspace_bytes, void* stream);

/* Latency path: encode calls with at most `max_tokens` packed tokens (0 = never, the default) run on
 * kernels shaped for ONE proof state — the reference's per-state call (`retrieve`,
 * retrieval/model.py:348-357) — instead of the 128 x 128 tiles that are sized for re-indexing: narrow
 * GEMM tiles (64 or 128 tokens x 64 columns, 128 x 128 for the gated FFN-up) that spread the state's work
 * over most of the SMs, the next layer's weights prefetched into L2 by the idle SMs, pooling as per-group
 * partial rows, everything chained by programmatic dependent launch.  Results agree with the
 * throughput path to a few 1e-4 on unit-norm embeddings (the RMSNorm statistics are summed in another
 * grouping, which flips the odd bf16 rounding of an intermediate), not bit for bit, so a caller that needs
 * re-indexing's bits leaves it off; within the latency path a sequence's embedding does not depend on what
 * else is in the call. */
int rpx_encoder_set_latency_tokens(rpx_encoder* enc, int32_t max_tokens);

/* T5 bidirectional relative-position bucket of `relative_position` = key - query
 * (HF modeling_t5.py:189-234).  Pure host function (no GPU needed); exported so the
 * CPU test-suite can pin the table the attention kernel uses against the HF code. */
int32_t rpx_t5_relative_bucket(int32_t relative_position, int32_t num_buckets, int32_t max_distance);

/* The unidirectional bucket the decoder's self-attention uses (HF `_relative_position_bucket(bidirectional=False)`):
 * relative_position = key - query <= 0 spreads over all `num_buckets`, positive positions fall in bucket 0.  Requires
 * max_distance > num_buckets / 2.  Pure host function. */
int32_t rpx_t5_relative_bucket_unidirectional(int32_t relative_position, int32_t num_buckets, int32_t max_distance);

/* Debug / parity hook: when non-NULL, every encode call also writes the fp32
 * residual stream after the embedding and after each block to
 * d_hidden[(layer) * n_tokens * d_model ...] (num_layers + 1 slabs, packed tokens). */
int rpx_encoder_set_debug_hidden(rpx_encoder* enc, float* d_hidden);

/* Per-kernel-class device timing (CUDA events on the launch stream).  Classes:
 * 0 embed, 1 qkv gemm, 2 attention, 3 o-proj gemm, 4 ffn-up gemm, 5 ffn-down gemm, 6 pool. */
#define RPX_N_KERNEL_CLASSES 7
int rpx_encoder_set_profiling(rpx_encoder* enc, int32_t enable);
/* Synchronises the recorded events; adds elapsed ms / launch counts since the
 * last read into ms[RPX_N_KERNEL_CLASSES], launches[RPX_N_KERNEL_CLASSES]. */
int rpx_encoder_read_profile(rpx_encoder* enc, float* h_ms, int64_t* h_launches);

/* ------------------------------------------------------------------- tactic generator
 * The teacher-forced forward of the reference's tactic generator, a `T5ForConditionalGeneration` (ByT5-small:
 * 12 encoder and 4 decoder layers):
 *     self.generator(input_ids=state_ids, attention_mask=state_mask, labels=tactic_ids)   generation/model.py:101-111
 * giving `.loss` and `.logits`.  The encoder half runs on an rpx_encoder built from the same checkpoint's
 * `encoder.*` keys; the decoder handle holds the decoder layers, the cross-attention K / V projections of all of
 * them and the output head.  Weights are packed as the encoder's are (bf16, each RMSNorm weight folded into the B
 * operand of the GEMM that follows it, FFN-up interleaved in 128-row blocks); in addition
 *   - the cross K / V weights of all decoder layers form one [num_layers * 2 * heads * d_kv, d_model] matrix with
 *     encoder.final_layer_norm folded in, applied once per call to the encoder's last residual stream;
 *   - decoder.final_layer_norm (and, with scale_decoder_outputs, d_model ** -0.5) is folded into the head rows.
 * HF key of each member on the right (i = decoder layer). */
typedef struct {
  const float* d_shared;         /* shared.weight (the decoder's embedding)                      [vocab, d_model] */
  const float* d_rel_bias;       /* decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight [buckets, heads] */
  const float* d_final_ln;       /* decoder.final_layer_norm.weight                              [d_model]        */
  const float* d_enc_final_ln;   /* encoder.final_layer_norm.weight                              [d_model]        */
  const float* d_head;           /* lm_head.weight, or shared.weight when the embeddings are tied [vocab, d_model] */
  const float* const* h_q;       /* decoder.block.i.layer.0.SelfAttention.q.weight               [heads*d_kv, d_model] */
  const float* const* h_k;       /* ...k.weight                                                                    */
  const float* const* h_v;       /* ...v.weight                                                                    */
  const float* const* h_o;       /* ...o.weight                                                  [d_model, heads*d_kv] */
  const float* const* h_ln0;     /* decoder.block.i.layer.0.layer_norm.weight                    [d_model]        */
  const float* const* h_cq;      /* decoder.block.i.layer.1.EncDecAttention.q.weight             [heads*d_kv, d_model] */
  const float* const* h_ck;      /* ...k.weight                                                                    */
  const float* const* h_cv;      /* ...v.weight                                                                    */
  const float* const* h_co;      /* ...o.weight                                                  [d_model, heads*d_kv] */
  const float* const* h_ln1;     /* decoder.block.i.layer.1.layer_norm.weight                    [d_model]        */
  const float* const* h_wi0;     /* decoder.block.i.layer.2.DenseReluDense.wi_0.weight           [d_ff, d_model]  */
  const float* const* h_wi1;     /* ...wi_1.weight                                                                 */
  const float* const* h_wo;      /* ...wo.weight                                                 [d_model, d_ff]  */
  const float* const* h_ln2;     /* decoder.block.i.layer.2.layer_norm.weight                    [d_model]        */
} rpx_t5_decoder_weights;

typedef struct rpx_t5_decoder rpx_t5_decoder; /* opaque */

/* `cfg` describes the decoder: num_layers = the checkpoint's num_decoder_layers, everything else as the encoder's.
 * 0 for a config rpx_t5_decoder_create rejects. */
size_t rpx_t5_decoder_packed_bytes(const rpx_t5_config* cfg);
/* Packs the weights into d_packed (synchronises `stream`; the fp32 weights may be freed on return).
 *   scale_decoder_outputs  nonzero: logits are scaled by d_model ** -0.5 (HF T5 with tied embeddings)
 *   start_token_id         decoder_start_token_id, which must equal the pad id (HF `_shift_right` feeds both) */
int rpx_t5_decoder_create(const rpx_t5_config* cfg, const rpx_t5_decoder_weights* w, int32_t scale_decoder_outputs,
                          int32_t start_token_id, void* d_packed, size_t packed_bytes, void* stream,
                          rpx_t5_decoder** out);
int rpx_t5_decoder_destroy(rpx_t5_decoder* dec);

/* Workspace of one rpx_seq2seq_forward call on [batch, in_len] states and [batch, out_len] labels (0 when `dec`
 * and `enc` do not fit together). */
size_t rpx_seq2seq_workspace_bytes(const rpx_t5_decoder* dec, const rpx_encoder* enc, int32_t batch, int32_t in_len,
                                   int32_t out_len);
/* HF `T5ForConditionalGeneration(input_ids, attention_mask, labels)` (teacher forcing), on the throughput tiles:
 *   d_input_ids       int64 [batch, in_len] state ids; d_attention_mask int64 [batch, in_len] right-padded prefix mask
 *                     with at least one token per row (RPX_ERR_MASK otherwise), or NULL: every position is a token
 *   d_labels          int64 [batch, out_len]: target ids in [0, vocab) or -100 (ignored)
 *   d_logits          optional fp32 [batch, out_len, vocab]
 *   d_seq_logprob     fp64 [batch]: sum over the counted positions of log_softmax(logits)[label]
 *   d_seq_count       int32 [batch]: the counted positions (labels != -100)
 * Decoder inputs are HF `_shift_right(labels)`: start token, then labels[:, :-1] with -100 fed as the pad id.  Row
 * b's decoder length is the last position whose label is not -100, plus one; positions at or past it are never
 * computed (causality: no counted position sees them) and their logits are written as zeros, where HF computes
 * values that its loss ignores.  HF's loss is -sum(seq_logprob) / sum(seq_count).  Every output row depends on its
 * own row of the inputs alone.  Ids outside [0, vocab) in d_input_ids give RPX_ERR_INVALID (after the call ran
 * with id 0 in their place); labels that are neither -100 nor in [0, vocab) give RPX_ERR_INVALID before anything
 * runs.  Synchronises `stream` twice (lengths, then the id check). */
int rpx_seq2seq_forward(rpx_t5_decoder* dec, rpx_encoder* enc, const int64_t* d_input_ids,
                        const int64_t* d_attention_mask, int32_t batch, int32_t in_len, const int64_t* d_labels,
                        int32_t out_len, float* d_logits, double* d_seq_logprob, int32_t* d_seq_count,
                        void* d_workspace, size_t workspace_bytes, void* stream);

/* Workspace of one rpx_seq2seq_generate call (0 when the arguments are out of range or `dec` and `enc` do not fit
 * together).  Dominated by the KV cache: num_layers * max_length * batch * num_beams * 3 * inner bf16. */
size_t rpx_seq2seq_generate_workspace_bytes(const rpx_t5_decoder* dec, const rpx_encoder* enc, int32_t batch,
                                            int32_t in_len, int32_t num_beams, int32_t max_length);
/* Optional record of every step of a generate call, for tests: step t (t < max_steps) writes
 *   d_scores   [max_steps][R][vocab] fp32  the step's log-probs (num_beams == 1: the logits), R = batch * num_beams
 *   d_parents  [max_steps][R] int32        the row each next-step row continues (global row)
 *   d_tokens   [max_steps][R] int32        the token each next-step row appends
 * Rows of a state whose search has ended are not written. */
typedef struct rpx_generate_trace {
  float* d_scores;
  int32_t* d_parents;
  int32_t* d_tokens;
  int32_t max_steps;
} rpx_generate_trace;
/* HF `T5ForConditionalGeneration.generate(input_ids, attention_mask, num_beams, num_return_sequences, max_length,
 * length_penalty, do_sample=False, early_stopping=False)` with one EOS id and no logits processor: HF 5.5's
 * `_beam_search` (num_beams > 1) or greedy `_sample` (num_beams == 1), each state's beams decoded together over a KV
 * cache, every search step on the device.
 *   d_input_ids / d_attention_mask  as rpx_seq2seq_forward (the mask may be NULL: every position is a token)
 *   d_sequences  int64 [batch * num_return, max_length]: row b * num_return + j is state b's j-th best hypothesis,
 *                the decoder start id, its tokens, then the fill id (beam: pad id, or eos_id when the pad id is 0, as
 *                HF's `output_fill_value`; greedy: the pad id).  Columns [0, *h_out_len) are HF's `sequences`.
 *   d_scores     fp32 [batch * num_return]: HF's `sequences_scores` (beam search only; may be NULL for greedy)
 *   h_out_len    host: 1 + the longest returned hypothesis;  h_steps (host, optional): the decoder steps HF runs
 *                for this call (the step at which the last search ended).  The engine checks for completion every 8
 *                steps, so it may run up to 15 more steps whose GEMMs do full work and change no result.
 * Candidates are ranked by score, ties by flat index (beam * vocab + token) ascending.  Checks: 1 <= num_return <=
 * num_beams <= 128, 2 num_beams <= vocab_size (beam search), max_length >= 2, eos_id in the vocabulary; a bad mask
 * gives RPX_ERR_MASK, ids outside the vocabulary RPX_ERR_INVALID.  Synchronises `stream`. */
int rpx_seq2seq_generate(rpx_t5_decoder* dec, rpx_encoder* enc, const int64_t* d_input_ids,
                         const int64_t* d_attention_mask, int32_t batch, int32_t in_len, int32_t num_beams,
                         int32_t num_return, int32_t max_length, double length_penalty, int32_t eos_id,
                         int64_t* d_sequences, float* d_scores, int32_t* h_out_len, int32_t* h_steps,
                         const rpx_generate_trace* trace, void* d_workspace, size_t workspace_bytes, void* stream);

/* Workspace of one rpx_seq2seq_evaluate call (0 when the arguments are out of range or `dec` and `enc` do not fit
 * together): one prefill, and the larger of the two halves' own regions, which they share. */
size_t rpx_seq2seq_evaluate_workspace_bytes(const rpx_t5_decoder* dec, const rpx_encoder* enc, int32_t batch,
                                            int32_t in_len, int32_t out_len, int32_t num_beams, int32_t max_length);
/* rpx_seq2seq_forward and rpx_seq2seq_generate on the same states, as the reference's `validation_step` runs the loss
 * and `generate` on one batch, with the encoder and the cross K / V computed once for both.  Every argument means what
 * it means in those two calls, and each output equals theirs bit for bit.  The checks are those of both calls; the
 * label check comes before anything runs, the id check once after both halves.  Synchronises `stream`. */
int rpx_seq2seq_evaluate(rpx_t5_decoder* dec, rpx_encoder* enc, const int64_t* d_input_ids,
                         const int64_t* d_attention_mask, int32_t batch, int32_t in_len, const int64_t* d_labels,
                         int32_t out_len, float* d_logits, double* d_seq_logprob, int32_t* d_seq_count,
                         int32_t num_beams, int32_t num_return, int32_t max_length, double length_penalty,
                         int32_t eos_id, int64_t* d_sequences, float* d_scores, int32_t* h_out_len, int32_t* h_steps,
                         void* d_workspace, size_t workspace_bytes, void* stream);

/* --------------------------------------------------------------- similarity + top-k
 * Replaces the matmul + argsort half of `Corpus.get_nearest_premises`
 * (common.py:307-308) and the first-k walk at :316-322:
 *     S = Q E^T ; per query the k best rows of E, best first.
 * Ordering contract (deterministic refinement of the reference's unspecified
 * argsort tie order): score descending, then index ascending, where `score` is
 * the canonical fp64 dot product of the bf16 operands (oracle/rpx_oracle.c:
 * rpx_oracle_dot64).  out_scores are that value rounded to fp32.
 *
 * Exactness.  The fast paths rank by an fp32 score (tensor-core or FMA accumulation)
 * and re-score a superset of the answer in fp64.  A per-query guard compares the k-th
 * re-scored entry with the best fp32 score any row outside the re-scored set can have;
 * when the gap is inside the accumulation error bound (c(d) * ||q|| * max_i ||e_i||)
 * the query is recomputed by an exact fp64 pass over all admissible rows.  The result is
 * therefore the contract's answer on any input (near-duplicate rows included); only the
 * time depends on the data.
 *
 * rpx_index — a handle on a [n, d] bf16 matrix (what the reference keeps in
 * `self.corpus_embeddings`, retrieval/model.py:190, 363-366; d % 64 == 0).  Creating it
 * runs the one pass that depends only on the matrix (row-norm bound of the guard).  The
 * caller owns the matrix and the `rpx_index_state_bytes()` bytes of device state it hands in;
 * both must outlive the handle, and the handle must be re-created after the matrix changes.
 * One call at a time per handle (the device state holds the call's counters).
 */
typedef struct rpx_index rpx_index; /* opaque */
size_t rpx_index_state_bytes(void);
int rpx_index_create(const void* d_E, int64_t n, int32_t d, void* d_state, void* stream, rpx_index** out);
int rpx_index_destroy(rpx_index* ix);
/* Diagnostics (synchronises `stream`): the row-norm bound, the largest |fp32 - fp64| score difference
 * and the largest epsilon any guard has seen, and how many queries took the exact pass. */
int rpx_index_stats(rpx_index* ix, void* stream, float* h_norm_max, float* h_max_err, float* h_max_eps,
                    int64_t* h_n_exact);

/* Path selection flags of rpx_index_topk (0 = automatic: streaming kernel for nq <= 2, tensor-core
 * kernel otherwise, exact pass for k > 200).  The forcing flags exist for parity tests; forced
 * streaming takes 1-2 queries (RPX_ERR_UNSUPPORTED otherwise). */
enum { RPX_TOPK_AUTO = 0, RPX_TOPK_FORCE_MMA = 1, RPX_TOPK_FORCE_STREAM = 2, RPX_TOPK_FORCE_EXACT = 4 };

/*   d_Q [nq, d] bf16; 1 <= k <= 1024 (k <= 200 on the fast paths).
 *   d_access_mask  optional bitmask, row q = mask_stride_words uint32 words, bit
 *                  (i & 31) of word i >> 5 set <=> premise i is accessible to query q
 *                  (the `p in accessible_premises` test, common.py:313-318).
 *   d_out_count    optional [nq]: number of valid results (< k when fewer than k
 *                  candidates exist; the tail is idx = -1, score = -inf).
 *   d_out_scores64 optional [nq, k] fp64 scores.
 *   d_out_packed   optional [nq, k, 2] int64: (fp64 score bits, index) records — the
 *                  payload of the multi-GPU all-gather (rpx_topk_merge_packed).
 *   idx_offset     added to every output index (row offset of this shard).
 */
size_t rpx_index_topk_workspace_bytes(int64_t n, int32_t d, int32_t nq, int32_t k);
int rpx_index_topk(rpx_index* ix, const void* d_Q, int32_t nq, int32_t k, const uint32_t* d_access_mask,
                   int64_t mask_stride_words, float* d_out_scores, double* d_out_scores64, int64_t* d_out_idx,
                   int32_t* d_out_count, int64_t* d_out_packed, int64_t idx_offset, int32_t flags,
                   void* d_workspace, size_t workspace_bytes, void* stream);

/* One-shot form without a handle: same result, but the row-norm pass over E runs on every call
 * (one extra read of the matrix).  Use rpx_index_* when the same matrix is queried repeatedly. */
size_t rpx_sim_topk_workspace_bytes(int64_t n, int32_t d, int32_t nq, int32_t k);
int rpx_sim_topk(const void* d_Q, int32_t nq, const void* d_E, int64_t n, int32_t d, int32_t k,
                 const uint32_t* d_access_mask, int64_t mask_stride_words, float* d_out_scores,
                 double* d_out_scores64, int64_t* d_out_idx, int32_t* d_out_count,
                 int64_t idx_offset, void* d_workspace, size_t workspace_bytes, void* stream);

/* k-way merge of per-shard results after the all-gather (SURVEY.md §8e):
 * inputs [n_parts, nq, k] (fp64 scores, int64 global indices; each [part, query] row sorted under
 * the ordering contract with its empty slots, idx < 0, at the end — exactly what the top-k calls
 * emit), outputs the global top-k per query under the same ordering contract.
 * The _packed form takes the gathered `d_out_packed` records, [n_parts, nq, k, 2] int64. */
int rpx_topk_merge(const double* d_scores64, const int64_t* d_idx, int32_t n_parts, int32_t nq,
                   int32_t k, float* d_out_scores, double* d_out_scores64, int64_t* d_out_idx,
                   int32_t* d_out_count, void* stream);
int rpx_topk_merge_packed(const int64_t* d_packed, int32_t n_parts, int32_t nq, int32_t k,
                          float* d_out_scores, double* d_out_scores64, int64_t* d_out_idx,
                          int32_t* d_out_count, void* stream);

/* ------------------------------------------------------------------------------ BM25
 * Replaces the scoring and ranking of the reference's BM25 baseline (retrieval/bm25/main.py:48-52):
 *     scores = bm25.get_batch_scores(query_tokens, accessible);  np.argsort(scores)[::-1][:num_retrieved]
 * with rank_bm25.BM25Okapi's arithmetic.  The index is an inverted index in CSR form, built on the host
 * (reprover_b200/bm25.py) and owned by the caller:
 *   d_term_ptr  [vocab + 1] int64  the postings of term t are [term_ptr[t], term_ptr[t + 1])
 *   d_post_doc  [nnz] int32        document (premise) index, strictly ascending within a term
 *   d_post_c    [nnz] fp64         the term's contribution to that document's score,
 *                                  idf[t] * (tf * 2.5 / (tf + 1.5 * (0.25 + 0.75 * doc_len / avgdl)))
 * A query is a list of term ids in query order, repeats included; an id outside [0, vocab) adds nothing, like a token
 * the corpus does not contain.  A document's score is the fp64 sum ((0 + c(q1, d)) + c(q2, d)) + ... over the query
 * tokens present in it, added in query order, so it equals get_batch_scores bit for bit.  Ranking: score descending,
 * then index ascending (the reference's argsort leaves ties in no defined order).
 */
typedef struct rpx_bm25 rpx_bm25; /* opaque; the arrays must outlive it */
int rpx_bm25_create(const int64_t* d_term_ptr, const int32_t* d_post_doc, const double* d_post_c, int32_t vocab,
                    int64_t n_docs, int64_t nnz, rpx_bm25** out);
int rpx_bm25_destroy(rpx_bm25* ix);
/* 0 when the request is out of range (nq outside [1, 65535], k outside [1, 1024]). */
size_t rpx_bm25_topk_workspace_bytes(int64_t n_docs, int32_t nq, int32_t k);
/* The k best accessible documents of each of nq queries.
 *   d_tokens       concatenated term ids of all queries (device)
 *   h_offsets      nq + 1 non-decreasing offsets into d_tokens (HOST)
 *   d_access_mask  optional [n_mask_rows][mask_stride_words] uint32 bitmask in rpx_index_topk's layout; query q uses
 *                  row h_mask_rows[q] (HOST), so the queries of one theorem can share a row.  NULL: every document.
 *   d_out_scores64, d_out_idx  [nq, k]; d_out_count optional [nq] = min(k, accessible documents).  Slots past the
 *                  count hold score -inf, index -1.
 * The host arrays are copied before the call returns.  One query's result does not depend on the others in the call. */
int rpx_bm25_topk(const rpx_bm25* ix, const int32_t* d_tokens, const int64_t* h_offsets, int32_t nq,
                  const uint32_t* d_access_mask, int64_t mask_stride_words, const int32_t* h_mask_rows,
                  int32_t n_mask_rows, int32_t k, double* d_out_scores64, int64_t* d_out_idx, int32_t* d_out_count,
                  void* d_workspace, size_t workspace_bytes, void* stream);
/* get_batch_scores over every document: d_out [n_docs] fp64 scores of the one query d_tokens[0, n_tokens). */
int rpx_bm25_scores(const rpx_bm25* ix, const int32_t* d_tokens, int64_t n_tokens, double* d_out, void* stream);

/* ------------------------------------------------------------------- test utilities
 * Debug timeline: while `d_stamps` (device, n_slots x 8 uint64) is set, every launch of the 1-CTA GEMM
 * kernel takes the next slot and its CTA 0 records %globaltimer at: kernel entry, prologue done,
 * producer past the dependency wait, first operand stage landed, last MMA committed, accumulator seen by
 * the epilogue, epilogue done, kernel exit.  NULL switches it off.  Not thread-safe; tooling only. */
int rpx_debug_set_timeline(unsigned long long* d_stamps, int32_t n_slots);

/*
 * Plain wgmma GEMM used by the parity tests of the contraction core:
 * C[M, N] (fp32, ldc = N) = A[M, K] * B[N, K]^T, bf16 inputs; K % 64 == 0, N % 32 == 0. */
int rpx_gemm_bf16_f32(const void* d_A, const void* d_B, float* d_C, int32_t M, int32_t N,
                      int32_t K, void* stream);
/* Same contract through the 128 x 128 tiles of the core that runs QKV on the throughput path, every GEMM
 * of the latency path and the similarity stages of the top-k. */
int rpx_gemm1_bf16_f32(const void* d_A, const void* d_B, float* d_C, int32_t M, int32_t N,
                       int32_t K, void* stream);

enum { RPX_EGEMM_QKV = 0, RPX_EGEMM_OPROJ = 1, RPX_EGEMM_FFN_UP = 2, RPX_EGEMM_FFN_DOWN = 3, RPX_EGEMM_HEAD = 4 };
/* One encoder GEMM, launched as the forward pass launches it for T tokens on the throughput (latency = 0) or
 * latency path, PDL scope set as forward() sets it for that T.  A [T, K] bf16 (lda = K), B [N, K] bf16 in the
 * packed layout rpx_encoder_create writes.  D = d_model = K for QKV / FFN-up / HEAD, N for O-proj / FFN-down.
 *   QKV     out [T, N] bf16 = bf16(A B^T * rs[m]),  rs from ss_in
 *   FFN_UP  out [T, N/2] bf16 gated GELU,             rs from ss_in;  N % 256 == 0
 *   OPROJ / FFN_DOWN   h32 [T, N] += A B^T;  h16 = bf16(h32);  ss_out partials
 *   HEAD    out [T, N] fp32 = A B^T * rs[m], the generator's output head, rs from ss_in;  N % 32 == 0.  It runs on
 *           the throughput core on both paths (as in the teacher-forced forward and in every decode step);
 *           `latency` selects only the layout of ss_in.
 * ss_in / ss_out: [parts][T] fp32, parts = ceil(D / 128) (throughput) or D / 32 (latency).
 * d_prefetch (latency QKV only, else NULL): prefetch_bytes fetched into L2 by the CTAs the GEMM leaves idle. */
int rpx_debug_encoder_gemm(int32_t site, int32_t latency, const void* d_A, const void* d_B, int32_t T,
                           int32_t N, int32_t K, float ln_eps, const float* d_ss_in, void* d_out,
                           float* d_h32, void* d_h16, float* d_ss_out, const void* d_prefetch,
                           size_t prefetch_bytes, void* stream);

/* The relative-position bias table of the attention kernel, built as rpx_encoder_create builds it:
 * d_lut [n_heads][2 R + 1] fp32 (R = rel_max_distance), lut[h][delta + R] = d_rel_bias[bucket(delta)][h] for
 * delta = key - query, from an HF-layout relative_attention_bias table d_rel_bias [rel_buckets][n_heads] fp32.
 * Rejects the configs rpx_encoder_create rejects.  Synchronises `stream`; stages the (2 R + 1)-entry bucket
 * table in a stream-ordered allocation it frees before returning. */
int rpx_debug_attention_lut(const float* d_rel_bias, int32_t n_heads, int32_t rel_buckets,
                            int32_t rel_max_distance, float* d_lut, void* stream);
/* The encoder's attention, launched as the forward pass launches it for n_tokens tokens on the throughput
 * (latency = 0) or latency path, PDL scope set as forward() sets it.
 *   d_qkv   [n_tokens, 3 * n_heads * 64] bf16: q | k | v, head h in columns [64 h, 64 h + 64) of each
 *   d_out   [n_tokens, n_heads * 64] bf16; rows of tokens outside every sequence are not written
 *   d_cu_seqlens  [n_seqs + 1] int32 token offsets of the packed sequences on the device; the caller
 *           guarantees 0 = cu[0] < cu[1] < ... < cu[n_seqs] <= n_tokens and max_len >= every length
 *   d_lut   from rpx_debug_attention_lut with the same n_heads and rel_max_distance
 * 1 <= n_seqs <= 65535 (the grid limit; more returns RPX_ERR_UNSUPPORTED).  Does not synchronise. */
int rpx_debug_attention(int32_t latency, const void* d_qkv, void* d_out, const int32_t* d_cu_seqlens,
                        const float* d_lut, int32_t n_tokens, int32_t n_seqs, int32_t max_len,
                        int32_t n_heads, int32_t rel_max_distance, void* stream);

/* rpx_debug_attention_lut with the bucket direction chosen: bidirectional != 0 is the encoder's table, 0 the
 * decoder's (unidirectional buckets; requires rel_max_distance > rel_buckets / 2). */
int rpx_debug_attention_lut_ex(const float* d_rel_bias, int32_t n_heads, int32_t rel_buckets,
                               int32_t rel_max_distance, int32_t bidirectional, float* d_lut, void* stream);
enum { RPX_ATTN_BIDIRECTIONAL = 0, RPX_ATTN_CAUSAL = 1, RPX_ATTN_CROSS = 2 };
/* The attention kernel in any of its modes, launched as the generator's forward launches it (throughput PDL
 * scope for n_q_tokens).
 *   RPX_ATTN_BIDIRECTIONAL, RPX_ATTN_CAUSAL  d_q = qkv [n_q_tokens, 3 * n_heads * 64] as rpx_debug_attention; d_kv and
 *           d_cu_kv are ignored (NULL); causal: key j visible to query i iff j <= i
 *   RPX_ATTN_CROSS  d_q [n_q_tokens, n_heads * 64] queries; d_kv [n_kv_tokens, 2 * n_heads * 64] k | v with its own
 *           d_cu_kv [n_seqs + 1]; every query of sequence s sees all keys of sequence s; no bias, d_lut ignored
 *   d_out   [n_q_tokens, n_heads * 64] bf16; max_len >= every query sequence's length.  Does not synchronise. */
int rpx_debug_attention_ex(int32_t mode, const void* d_q, const void* d_kv, void* d_out, const int32_t* d_cu_q,
                           const int32_t* d_cu_kv, const float* d_lut, int32_t n_q_tokens, int32_t n_kv_tokens,
                           int32_t n_seqs, int32_t max_len, int32_t n_heads, int32_t rel_max_distance, void* stream);

/* The generator's decode self-attention at step t, as rpx_seq2seq_generate launches it:
 *   d_cache  [max_length][rows][3 * n_heads * 64] bf16 (q | k | v); query of row r: cache row t * rows + r
 *   d_lin    [rows][max_length] int32: key / value p of row r (p = 0..t) is cache row p * rows + lin[r][p]; NULL: r
 *   d_lut    the decoder's table (rpx_debug_attention_lut_ex, bidirectional = 0)
 *   d_out    [rows, n_heads * 64] bf16 = softmax_p(q.k_p + lut[h][max(p - t, -R) + R]) v_p per head, unscaled.
 * Does not synchronise. */
int rpx_debug_decode_attention(const void* d_cache, const int32_t* d_lin, const float* d_lut, void* d_out, int32_t t,
                               int32_t rows, int32_t max_length, int32_t n_heads, int32_t rel_max_distance,
                               void* stream);

/* The search half of rpx_seq2seq_generate on caller-supplied logits, for tests: the same init, step and finish
 * kernels with the same arguments, under the same checks (vocab in place of the decoder's vocab_size), with no
 * decoder or encoder.
 *   d_logits  fp32 [max_length - 1][batch * num_beams][vocab]: step t reads slab t as the decoder's logits of the
 *             rows' current tokens (row b * num_beams + j is beam j of state b)
 *   start_id  the decoder start id (also the pad id, as rpx_t5_decoder_create requires)
 * Outputs and the optional trace are those of rpx_seq2seq_generate; *h_steps is the step at which the last search
 * ended.  Every step runs (a state whose search is done returns at once from each later one).  Synchronises
 * `stream`. */
size_t rpx_debug_search_workspace_bytes(int32_t batch, int32_t num_beams, int32_t max_length);
int rpx_debug_search(const float* d_logits, int32_t batch, int32_t num_beams, int32_t vocab, int32_t num_return,
                     int32_t max_length, double length_penalty, int32_t eos_id, int32_t start_id,
                     int64_t* d_sequences, float* d_scores, int32_t* h_out_len, int32_t* h_steps,
                     const rpx_generate_trace* trace, void* d_workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RPX_H_ */
