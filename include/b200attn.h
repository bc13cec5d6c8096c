/*
 * b200attn.h -- C ABI of the H100-native paged-attention backend for mini-sglang.
 *
 * One shared library (libb200attn.so, built by mini-sglang_b200/build.py with
 * `nvcc -gencode arch=compute_90a,code=sm_90a`), plain pointers and sizes, no torch
 * types.  Every entry point enqueues work on the CUDA stream it is given and returns
 * immediately (never synchronises, CUDA-graph capturable).  Device pointers unless noted.
 *
 * Return value: 0 = OK, non-zero = error; b200_last_error() returns a thread-local
 * message.  The Python host turns a non-zero return into RuntimeError, mirroring the
 * reference's PanicError -> RuntimeError convention
 * (python/minisgl/kernel/csrc/include/minisgl/utils.h:40-88).
 *
 * Citations are path:line under the reference tree (M/ = python/minisgl/).
 * dtype codes: 0 = bfloat16, 1 = float16 (elementwise/store ops); attention is bf16/fp16.
 */
#ifndef B200ATTN_H_
#define B200ATTN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200_API __attribute__((visibility("default")))
#else
#define B200_API
#endif

#define B200_DTYPE_BF16 0
#define B200_DTYPE_FP16 1

/* ABI version of this header (bumped on any signature change). */
B200_API int b200_abi_version(void);
/* sha256 of the sources + flags this binary was built from (mini-sglang_b200/build.py compares it with
 * the tree to decide whether a rebuild is needed; a stale binary can therefore never pass as current). */
B200_API const char* b200_build_digest(void);
/* Thread-local description of the last non-zero return. */
B200_API const char* b200_last_error(void);
/* Number of kernels this library has launched so far (bench.py's gpu_launches). */
B200_API uint64_t b200_launch_count(void);
/* 1 if the library was compiled for sm_90a and the current device is CC 9.x. */
B200_API int b200_device_supported(void);
/* Kernel selection knobs (debug / cross-checking only; defaults are the product path):
 *   "decode_impl": 1 = wgmma + TMA kernel (default), 0 = cp.async / CUDA-core kernel.
 *   "prefill_impl": 1 = wgmma kernel (default, needs prefill_plan), 0 = mma.sync bring-up kernel.
 *   "prefill_order": 0 (default) = prefill work items size-sorted, heaviest first; 1 = request-major.
 *   "decode_fused_combine": 1 (default) = the chunk that arrives last merges the split-KV partials inside
 *       the decode launch (no combine launch), 0 = separate combine launch, 2 = in-kernel exactly when the
 *       plan policy leaves the batch unsplit.
 *   "decode_early_kv": 1 (default) = a decode launch that is being captured into a CUDA graph lets its TMA
 *       producers stream K/V before the predecessor kernel has finished (programmatic dependent launch; the
 *       metadata and this layer's pool slice are not written inside the graph); 0 = always wait first.
 *   "decode_plan_target": when splitting, aim at target * CTA-hint / kv_heads (request, chunk) items (default 2).
 *   "decode_plan_nosplit": no split-KV once bs * kv_heads * 100 >= value * CTA-hint (default 75; 0 = always split).
 * Returns the previous value, or -1 for an unknown name. */
B200_API int b200_set_option(const char* name, int value);

/* ---------------------------------------------------------------------------------------
 * K1  KV append.  Replaces `store_cache(k_cache, v_cache, indices, k, v)`
 *     (M/kernel/store.py:30-42 -> M/kernel/csrc/jit/store.cu:28-53,59-121), called from
 *     MHAKVCache.store_kv (M/kvcache/mha_pool.py:45-56).
 *     k_cache[indices[t]] = k[t]; v_cache[indices[t]] = v[t], rows of `row_bytes` bytes
 *     (multiple of 16).  Strides in bytes.  indices int32 (idx64 = 0) or int64 (idx64 = 1).
 * ------------------------------------------------------------------------------------- */
B200_API int b200_store_kv(void* k_cache, void* v_cache, int64_t cache_row_stride_bytes,
                  const void* k, const void* v, int64_t input_row_stride_bytes,
                  const void* indices, int idx64, int64_t num_tokens, int64_t row_bytes,
                  void* stream);

/* ---------------------------------------------------------------------------------------
 * K2  Row gather (SURVEY 8f "next": embedding lookup and last-token gather).  Replaces
 *     `indexing(weights, indices, output=, vocab_range=)` (M/kernel/index.py:32-53 ->
 *     M/kernel/csrc/jit/index.cu:34-96; caller VocabParallelEmbedding.forward,
 *     M/layers/embedding.py:31-41) and `x[indices].contiguous()` (M/layers/embedding.py:92-94).
 *     out[t] = weights[indices[t]], rows of `row_bytes` bytes (multiple of 16), strides in bytes.
 *     vocab_length >= 0 selects the masked form: pos = indices[t] - vocab_start; rows with
 *     pos outside [0, vocab_length) are zero-filled (the reference's masked_index_kernel).
 *     vocab_length < 0: plain gather; like the reference, indices are not range-checked.
 * ------------------------------------------------------------------------------------- */
B200_API int b200_index_rows(const void* weights, int64_t weight_row_stride_bytes, const void* indices,
                    int idx64, int64_t num_indices, int64_t row_bytes, void* out,
                    int64_t out_row_stride_bytes, int64_t vocab_start, int64_t vocab_length,
                    void* stream);

/* ---------------------------------------------------------------------------------------
 * K7  RMSNorm.  Replaces flashinfer.rmsnorm(x, w, eps, out=...) at M/layers/norm.py:16-21
 *     and the per-head q/k norm at M/layers/attention.py:50-53.
 *     x viewed as [rows, heads, dim]: element (r,h,i) at x + r*x_row_stride + h*x_head_stride + i
 *     (strides in elements); plain 2-D input uses heads = 1.  out may alias x (in place).
 *     y = float(x) * rsqrt(mean(x^2) + eps) * float(w), one rounding.  dim % 8 == 0, dim <= 8192.
 * ------------------------------------------------------------------------------------- */
B200_API int b200_rmsnorm(void* out, const void* x, const void* weight, int64_t rows, int heads, int dim,
                 int64_t x_row_stride, int64_t x_head_stride, int64_t out_row_stride,
                 int64_t out_head_stride, float eps, int dtype, void* stream);

/* flashinfer.fused_add_rmsnorm(x, residual, w, eps) at M/layers/norm.py:32-38 (both in place):
 * s = x + residual (fp32); residual <- round(s); x <- round(s * rsqrt(mean(s^2)+eps) * w). */
B200_API int b200_fused_add_rmsnorm(void* x, void* residual, const void* weight, int64_t rows, int dim,
                           int64_t x_row_stride, int64_t res_row_stride, float eps, int dtype,
                           void* stream);

/* ---------------------------------------------------------------------------------------
 * K6  RoPE.  Replaces flashinfer.apply_rope_with_cos_sin_cache_inplace(positions, query, key,
 *     head_size, cos_sin_cache) at M/layers/rotary.py:45-51: neox layout, fp32 cache
 *     [max_pos, head_dim] = cos | sin, in place on q [nnz, hq, head_dim] / k [nnz, hkv, head_dim]
 *     (row strides in elements, heads contiguous).  positions int32 (pos64=0) or int64.
 * ------------------------------------------------------------------------------------- */
B200_API int b200_rope_neox_inplace(void* q, void* k, const void* positions, int pos64,
                           const float* cos_sin_cache, int64_t nnz, int hq, int hkv, int head_dim,
                           int64_t q_row_stride, int64_t k_row_stride, int dtype, void* stream);

/* Fused pre-attention: per-head q/k RMSNorm (weights may be NULL = skip) followed by neox
 * RoPE, in place, one launch.  Replaces the three launches of AttentionLayer.forward
 * (M/layers/attention.py:50-54). */
B200_API int b200_qknorm_rope_inplace(void* q, void* k, const void* q_weight, const void* k_weight,
                             float eps, const void* positions, int pos64,
                             const float* cos_sin_cache, int64_t nnz, int hq, int hkv,
                             int head_dim, int64_t q_row_stride, int64_t k_row_stride, int dtype,
                             void* stream);

/* ---------------------------------------------------------------------------------------
 * a2/a3/a4  Metadata on device.  Replaces the host loops of prepare_metadata
 *     (M/attention/fa.py:67-105, fi.py:190-225): from per-request triples
 *     req_info[bs][3] = (table_idx, cached_len, device_len) (int32; device memory or PINNED host memory,
 *     which the kernels read in place -- no host-to-device copy on the step's critical path) and the global
 *     token-granular page table (M/core.py:103-104) produce
 *       seq_lens[bs]            = device_len
 *       cu_seqlens_q[bs+1]      = exclusive cumsum(device_len - cached_len)
 *       cu_seqlens_k[bs+1]      = exclusive cumsum(device_len)
 *       slot_table[bs][slot_table_stride] : row r = page_table[table_idx_r][0:width]
 *       decode_plan[b200_decode_plan_ints(bs)] :
 *         {chunk_tokens, total_chunks, bs, 0, chunk_start[bs+1], order[total_chunks]}
 *         (split-KV work list for b200_attn_decode: request r owns chunks
 *          [chunk_start[r], chunk_start[r+1]) of chunk_tokens tokens each; order[] lists the
 *          (request, chunk) items largest first, entry = r | chunk << 16 | n_chunks << 20).
 *     width = number of table columns to copy (>= max device_len, <= both strides).
 *     num_ctas_hint = persistent grid size the decode kernel will use (0 = default).
 * ------------------------------------------------------------------------------------- */
B200_API size_t b200_decode_plan_ints(int bs); /* = 4 + (bs + 1) + 16 * bs */
B200_API int b200_build_metadata(const int32_t* req_info, int bs, const int32_t* page_table,
                        int64_t page_table_stride, int32_t* seq_lens, int32_t* cu_seqlens_q,
                        int32_t* cu_seqlens_k, int32_t* slot_table, int64_t slot_table_stride,
                        int width, int32_t* decode_plan, int num_kv_heads, int num_ctas_hint,
                        void* stream);

/* Prefill work list for b200_attn_prefill: prefill_plan[4 + capacity_items] =
 * {n_items, 0, 0, 0, item[...]}, item = r | q_tile << 16 for every 128-row query tile of every
 * request, heaviest (most KV tiles under the causal mask) first.  capacity_items must be
 * >= sum_r ceil(q_len_r / 128) (<= nnz / 128 + bs); n_items = -1 reports an undersized buffer. */
B200_API int b200_build_prefill_plan(const int32_t* req_info, int bs, int32_t* prefill_plan,
                                     int capacity_items, void* stream);

/* ---------------------------------------------------------------------------------------
 * a1  Attention forward.  Replace BaseAttnBackend.forward (M/attention/base.py:20-22; impls
 *     fi.py:176-188, fa.py:49-65, trtllm.py:49-89): append k,v at out_loc, then causal
 *     (bottom-right) softmax(q k^T * scale) v over each request's slots.
 *     q   [nnz, hq, head_dim]  element (t,h,i) at q + t*q_row_stride + h*head_dim + i
 *     k,v [nnz, hkv*head_dim]  row strides k_row_stride / v_row_stride (elements)
 *     k_cache/v_cache: one layer of the pool viewed [num_slots, hkv, head_dim], contiguous rows
 *       (M/kvcache/mha_pool.py:28-43); slot stride = hkv*head_dim elements; num_slots bounds the
 *       TMA tensor map (rows >= num_slots read as zeros).
 *     page_size: allocation granularity behind the slot table (Context.page_size, M/core.py:103):
 *       the slots of positions [j*page_size, (j+1)*page_size) of a request are consecutive
 *       (M/scheduler/cache.py:119-146).  1 = no contiguity is assumed.
 *     slot_table [bs][slot_table_stride] int32 token-granular slots, seq_lens[bs] = kv length
 *       INCLUDING the tokens appended by this call.
 *     out [nnz, hq, head_dim] contiguous.  head_dim must be 128.
 *     workspace: b200_attn_workspace_bytes(max_bs, hq) bytes, owned by the caller, may be
 *       shared across layers (stream ordered).  It must be ZERO-FILLED once before its first use
 *       (it holds the split-KV arrival counters, which every launch leaves at zero again).
 * ------------------------------------------------------------------------------------- */
B200_API size_t b200_attn_workspace_bytes(int max_bs, int hq, int head_dim);

/* Decode: one query token per request (nnz == bs), KV append fused into the same launch. */
B200_API int b200_attn_decode(const void* q, int64_t q_row_stride, const void* k, int64_t k_row_stride,
                     const void* v, int64_t v_row_stride, void* k_cache, void* v_cache,
                     int64_t num_slots, int page_size, const int32_t* out_loc, const int32_t* slot_table, int64_t slot_table_stride,
                     const int32_t* seq_lens, const int32_t* decode_plan, int bs, int hq, int hkv,
                     int head_dim, float scale, void* out, void* workspace, size_t workspace_bytes,
                     int dtype, void* stream);

/* Decode with the pre-attention sequence of AttentionLayer.forward (M/layers/attention.py:50-54: per-head
 * q-norm, k-norm, neox RoPE -- three launches in the reference) folded into the same launch: q and k are the
 * RAW rows of the qkv projection; the kernel norms + ropes them on the fly (arithmetic of
 * b200_qknorm_rope_inplace, bit for bit), appends the roped k row and v row at out_loc and attends.  q / k
 * are NOT modified in memory (nothing downstream of attention reads them, M/models/utils.py:118-123).
 * q_weight / k_weight may be NULL (models without qk-norm); positions int32 [bs]; cos_sin_cache fp32
 * [max_pos, 128] = cos | sin (M/layers/rotary.py:24-32).  Everything else as b200_attn_decode. */
B200_API int b200_attn_decode_fused(const void* q, int64_t q_row_stride, const void* k, int64_t k_row_stride,
                     const void* v, int64_t v_row_stride, const void* q_weight, const void* k_weight, float eps,
                     const int32_t* positions, const float* cos_sin_cache, void* k_cache, void* v_cache,
                     int64_t num_slots, int page_size, const int32_t* out_loc, const int32_t* slot_table,
                     int64_t slot_table_stride, const int32_t* seq_lens, const int32_t* decode_plan, int bs,
                     int hq, int hkv, int head_dim, float scale, void* out, void* workspace,
                     size_t workspace_bytes, int dtype, void* stream);

/* Prefill / extend: ragged query rows, cu_seqlens_q[bs+1]; request r has
 * q_len = cu_seqlens_q[r+1]-cu_seqlens_q[r] new tokens at kv positions
 * [seq_lens[r]-q_len, seq_lens[r]).  max_seqlen_q is a host-side upper bound (grid sizing).
 * prefill_plan: b200_build_prefill_plan output (work list of the wgmma kernel); NULL selects
 * the mma.sync bring-up kernel (as does b200_set_option("prefill_impl", 0)). */
B200_API int b200_attn_prefill(const void* q, int64_t q_row_stride, const void* k, int64_t k_row_stride,
                      const void* v, int64_t v_row_stride, void* k_cache, void* v_cache,
                      int64_t num_slots, int page_size, const int32_t* out_loc, const int32_t* slot_table,
                      int64_t slot_table_stride, const int32_t* seq_lens,
                      const int32_t* cu_seqlens_q, const int32_t* prefill_plan, int bs, int64_t nnz,
                      int max_seqlen_q, int hq,
                      int hkv, int head_dim, float scale, void* out, void* workspace,
                      size_t workspace_bytes, int dtype, void* stream);

/* ---------------------------------------------------------------------------------------
 * f4  Tensor-parallel all-reduce for decode-sized messages, optionally fused with the residual add +
 *     RMSNorm that consumes it.  Replaces PyNCCLCommunicator.all_reduce (M/kernel/pynccl.py:14-22 ->
 *     M/kernel/csrc/src/pynccl.cu:93-134: copy into the symmetric window, ncclAllReduce, copy back)
 *     behind the reference's communication plug-in point DistributedCommunicator.plugins
 *     (M/distributed/impl.py:60-97), called after o_proj / down_proj (M/layers/linear.py:102-106,
 *     122-126), and -- fused form -- the flashinfer.fused_add_rmsnorm that follows
 *     (M/layers/norm.py:32-38).  One-shot "push" algorithm over NVLink peer memory with the payload as its own
 *     arrival flag (negative zeros in x are sent as +0.0): see csrc/allreduce.cu.  Every rank must issue the
 *     same sequence of calls with the same shapes.
 *
 *     Set-up (host, once): each rank allocates a region of b200_ar_region_bytes(world, max_bytes)
 *     with b200_ar_alloc (initialised: sentinel-filled data, zero counters), exports it with b200_ar_ipc_handle (64 opaque bytes), the
 *     handles are exchanged by the caller (torch.distributed), peers are mapped with b200_ar_ipc_open,
 *     and b200_ar_create receives the `world` base pointers in rank order (bases[rank] = own region;
 *     opened_mask[i] != 0 marks pointers b200_ar_destroy must unmap).
 *
 *     b200_ar_allreduce: x [rows, dim] (row stride in elements), 16-bit floats, rows*dim*2 <= max_bytes.
 *       residual == weight == NULL:  out <- sum over ranks of x (fp32 accumulation in rank order, one
 *         rounding; identical bits on every rank); out may alias x.
 *       else:  y = that sum; residual <- round(y + residual); out <- round((y + residual) *
 *         rsqrt(mean((y + residual)^2) + eps) * weight)  == b200_fused_add_rmsnorm(y, residual, ...),
 *         bit for bit; out may alias x.
 *     Capturable in CUDA graphs (the launch epoch lives in device memory); never synchronises.
 * ------------------------------------------------------------------------------------- */
B200_API size_t b200_ar_region_bytes(int world, size_t max_bytes);
B200_API int b200_ar_alloc(size_t bytes, void** ptr);
B200_API int b200_ar_ipc_handle(void* ptr, void* handle64);
B200_API int b200_ar_ipc_open(const void* handle64, void** ptr);
B200_API int b200_ar_create(int rank, int world, void* const* bases, const int* opened_mask,
                            size_t max_bytes, void** comm);
B200_API int b200_ar_destroy(void* comm, int free_local);
B200_API size_t b200_ar_max_bytes(const void* comm);
B200_API int b200_ar_allreduce(void* comm, const void* x, int64_t x_row_stride, void* out,
                               int64_t out_row_stride, void* residual, int64_t res_row_stride,
                               const void* weight, int64_t rows, int dim, float eps, int dtype,
                               void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200ATTN_H_ */
