/* b2rl.h — C ABI of the H100-native learner-side replay path.
 *
 * The reference (seungju-k1m/Distributed_RL) is pure Python and defines no
 * FFI of its own; its boundary for this path is three duck-typed Python
 * surfaces (SURVEY.md §8b).  Every entry point below therefore cites the
 * reference *Python* interface it replaces (paths relative to the reference
 * root).  The Python mirrors in distributed_rl_b200/ bind these with ctypes
 * (INTEGRATION.md shows the stub a reference maintainer would add).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch types.
 *   - every function returns 0 on success, <0 on error; the message is
 *     available (per thread) from b2rl_last_error().
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it
 *     and is asynchronous w.r.t. the host unless stated otherwise.
 *   - pointers named *_dev are device pointers owned by the caller (e.g.
 *     torch tensors' data_ptr()); the library never frees them.
 *   - the sum-tree and the payload arrays are owned by the handle and freed
 *     by b2rl_replay_destroy().
 *   - one producer + one consumer thread may use a handle concurrently as
 *     long as they enqueue on the same stream (stream order replaces the
 *     reference's `lock` flag handshake, APE_X/ReplayMemory.py:151-160).
 */
#ifndef B2RL_H_
#define B2RL_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2RL_MAX_FIELDS 8
#define B2RL_OK 0
#define B2RL_ERR_INVALID (-1)
#define B2RL_ERR_CUDA (-2)
#define B2RL_ERR_NOMEM (-3)

typedef struct b2rl_replay b2rl_replay; /* opaque */

/* One replay shard: a ring of `capacity` slots, `n_fields` SoA payload arrays
 * (field f holds capacity x field_bytes[f] bytes) and an fp64 sum-tree + fp32
 * min-tree over the slot priorities.
 * Replaces the storage of baseline/PER.py:48-66 (`memory` list of pickled
 * records + `Tree.prior_torch`) and baseline/utils.py:328-333
 * (PrioritizedMemory: CompressedDeque + SumTree). */
typedef struct {
  int64_t capacity;                      /* slots; the tree is padded to 2^k */
  int32_t n_fields;                      /* 0..B2RL_MAX_FIELDS               */
  int32_t device;                        /* CUDA device ordinal              */
  int64_t field_bytes[B2RL_MAX_FIELDS];  /* bytes per slot of each field     */
} b2rl_replay_desc;

const char* b2rl_last_error(void);
int b2rl_version(void);

/* PER.__init__ (baseline/PER.py:49-66), PrioritizedMemory.__init__
 * (baseline/utils.py:329-332). */
int b2rl_replay_create(const b2rl_replay_desc* desc, b2rl_replay** out);
int b2rl_replay_destroy(b2rl_replay* h);

/* PER.__init__ (baseline/PER.py:49-66) with each field placed where it is read from: on_host[f] != 0 puts field f in
 * pinned, mapped host memory owned by the handle (cudaHostAlloc with cudaHostAllocMapped | cudaHostAllocPortable;
 * the kernels address it through cudaHostGetDevicePointer), every other field and the sum-tree in device memory.
 * Meant for the frames of R2D2 sequences (R2D2/ReplayMemory.py:70-88), which a step reads only for the sampled
 * sequences.  A host field's row must be a whole number of 16-byte units.  B2RL_ERR_NOMEM, with the size in the
 * message, when the pinned allocation fails.  on_host == NULL is b2rl_replay_create.
 * Host fields are never read by bulk async (TMA) copies: b2rl_replay_gather and b2rl_serve_fill copy their sampled rows
 * with 16-byte loads through the mapped pointer, from a few CTAs (B2RL_HOST_GATHER_CTAS, default 8).  Every write
 * into a host field is stream-ordered on the call's stream: push, copy_payload and ingest_pipelined take a host
 * field's rows from device memory (cudaMemcpyAsync) or from pinned host memory (a copy kernel), and refuse pageable
 * host memory before any work; fill_hash writes them with its kernel.  b2rl_dedup_attach and b2rl_serve_fill_uniform
 * refuse a handle with host fields. */
int b2rl_replay_create_placed(const b2rl_replay_desc* desc, const int32_t* on_host, b2rl_replay** out);
/* Where field f of PER.memory (baseline/PER.py:7-28) lives: *on_host = 1 for pinned host memory, 0 for device. */
int b2rl_replay_field_placement(const b2rl_replay* h, int32_t field, int32_t* on_host);

/* PER.__len__ (baseline/PER.py:80-81): number of valid slots, capacity, and
 * the ring head (next slot to be written). Host-side, no sync. */
int b2rl_replay_size(const b2rl_replay* h, int64_t* size, int64_t* capacity, int64_t* head);

/* Device base pointer of payload field f (capacity x field_bytes[f] bytes): the storage behind
 * PER.memory / Tree.data (baseline/PER.py:7-28), exposed so that consumers (b2rl_conv1_fused) read rows in place.
 * For a field placed on the host (b2rl_replay_create_placed) it is the HOST address of the pinned rows: never pass
 * it to b2rl_conv1_fused or b2rl_conv1_wgrad. */
int b2rl_replay_field_ptr(const b2rl_replay* h, int32_t field, void** ptr_dev);

/* PER.push (baseline/PER.py:69-75) / PrioritizedMemory.push
 * (baseline/utils.py:334-337): append n records.  fields_src[f] points to
 * n x field_bytes[f] contiguous bytes (host — ideally pinned — or device;
 * copied with cudaMemcpyDefault), prios to n fp32 priorities (same rule).
 * Slots are written at the ring head; when the ring is full the oldest slots
 * are overwritten (FIFO, as PER.remove_to_fit :118-127 drops them — but slot
 * ids stay stable instead of being renumbered).  Leaves and their root paths
 * are refreshed in the same call.  n <= capacity. */
int b2rl_replay_push(b2rl_replay* h, const void* const* fields_src, const float* prios,
                     int64_t n, void* stream);

/* Pipelined ingest — the same PER.push (baseline/PER.py:69-75; drained from Redis by Replay.run,
 * APE_X/ReplayMemory.py:128-139), split so that the host->device copy of the NEXT batch of
 * records can run on its own stream while the learner step of the current batch computes:
 *   reserve   (learner stream) priorities of the next n ring slots := 0, so the records about to
 *             be overwritten can no longer be sampled; *start_slot receives the first slot
 *   copy      (ingest stream, after an event recorded behind `reserve`) payload rows only
 *   commit    (learner stream, after the copy's event) priorities + root paths; advances the ring
 * reserve/commit must alternate; n <= capacity. */
int b2rl_replay_reserve(b2rl_replay* h, int64_t n, int64_t* start_slot, void* stream);
int b2rl_replay_copy_payload(b2rl_replay* h, const void* const* fields_src, int64_t start_slot, int64_t n,
                             void* stream);
int b2rl_replay_commit(b2rl_replay* h, const float* prios, int64_t n, void* stream);

/* The steady-state form of the ingest loop of Replay.run (APE_X/ReplayMemory.py:128-139: drain -> PER.push) as ONE
 * call per learner iteration: (1) the batch whose host->device copy the previous call started is published —
 * `stream` waits for that copy, then its priorities are written (PER.push's priority append, baseline/PER.py:69-75);
 * (2) the ring slots of the next batch are retired (priority 0: unsampleable while they are overwritten) and its
 * payload + priorities are copied on a library-owned copy stream, overlapping whatever is enqueued on `stream`
 * next.  Host buffers (pinned) must stay valid and unmodified until their copy has executed (the call is
 * asynchronous: synchronize `stream` after the NEXT call, or keep enough staging sets).  fields_src == NULL:
 * publish only (flush).
 * Do not interleave with b2rl_replay_reserve / b2rl_replay_commit. */
int b2rl_replay_ingest_pipelined(b2rl_replay* h, const void* const* fields_src, const float* prios_src, int64_t n,
                                 void* stream);

/* PER.remove_to_fit (baseline/PER.py:118-127): drop the `delta` oldest
 * records (priority := 0 so they can never be sampled; size -= delta). */
int b2rl_replay_evict(b2rl_replay* h, int64_t delta, void* stream);

/* Benchmark / property-test helper (no reference counterpart; stands in for a replay pre-filled through
 * PER.push, baseline/PER.py:69-75, with SURVEY.md §8d's synthetic frames): fill slots
 * [0, n) of every field with the counter hash documented in DESIGN.md §4
 * (word w of slot s of field f = lowbias32(seed ^ f*0x9E3779B9 ^ s*2654435761
 * ^ w*2246822519)) and mark them valid.  Priorities are NOT touched: follow
 * with b2rl_tree_build(). */
int b2rl_replay_fill_hash(b2rl_replay* h, int64_t n, uint32_t seed, void* stream);

/* Bulk (re)build: priorities of slots [0, n) := prios_dev[0..n), the rest 0,
 * then every internal node is recomputed (node = left + right in fp64, as
 * baseline/sumtree.py Node._reduce :21-27).  State equals
 * SumTree.extend(prios) (:97-99) / Tree.push (baseline/PER.py:22-28). */
int b2rl_tree_build(b2rl_replay* h, const float* prios_dev, int64_t n, void* stream);

/* PER.sample (baseline/PER.py:92-116) + the IS-weight lines of
 * APE_X/ReplayMemory.py:65-67 and PER.max_weight (:129-133), with the
 * descent rule of SumTree.prioritized_sample / Node._find
 * (baseline/sumtree.py:53-62,128-140): pos = root*u; at each node
 * `pos < left ? left : (pos -= left, right)`.
 *   u01_dev   n fp64 uniforms in [0,1) on the device, or NULL to draw them
 *             from Philox4x32-10 (seed, counter = rng_offset + k)
 *   idx_out   int64[n]  sampled slot ids (with replacement)
 *   prob_out  fp32[n]   p_i / sum(p)               (may be NULL)
 *   w_out     fp32[n]   (1/(N*prob))^beta / max_w  (may be NULL)
 *   max_w_dev NULL: max_w is this shard's own max_j (N*prob_j)^-beta.  Non-NULL:
 *             one device float used instead — the all-reduced MAX over the shards
 *             of a multi-GPU replay (SURVEY.md §8e "priority-max reduction").
 * Sampling from an empty tree is an error. */
int b2rl_tree_sample(b2rl_replay* h, const double* u01_dev, uint64_t seed, uint64_t rng_offset,
                     int64_t n, float beta, const float* max_w_dev, int64_t* idx_out_dev,
                     float* prob_out_dev, float* w_out_dev, void* stream);

/* Same (PER.sample, baseline/PER.py:92-116), but the uniforms come from the handle's DEVICE-RESIDENT Philox stream
 * {seed, counter} (set with b2rl_replay_seed), and the counter is advanced by n
 * on the stream afterwards — so the call can be captured in a CUDA graph and
 * every replay draws fresh numbers.  Draw k of the call uses counter + k. */
int b2rl_replay_seed(b2rl_replay* h, uint64_t seed, uint64_t counter, void* stream);
int b2rl_tree_sample_stream(b2rl_replay* h, int64_t n, float beta, const float* max_w_dev,
                            int64_t* idx_out_dev, float* prob_out_dev, float* w_out_dev, void* stream);

/* b2rl_tree_sample_stream + the part of Replay.buffer (APE_X/ReplayMemory.py:74-93) that unpacks the SCALAR
 * fields of the sampled records (action, reward, done): for every field f with small_fields_out_dev[f] != NULL
 * (field_bytes[f] must be 1, 2, 4 or 8) row idx[k] is copied to small_fields_out_dev[f] + k*field_bytes[f] by the
 * sampling thread itself, so a learner step needs no separate gather launch for them (the frame fields are read
 * in place by b2rl_conv1_fused).  small_fields_out_dev may be NULL (= b2rl_tree_sample_stream). */
int b2rl_tree_sample_fetch(b2rl_replay* h, int64_t n, float beta, const float* max_w_dev,
                           int64_t* idx_out_dev, float* prob_out_dev, float* w_out_dev,
                           void* const* small_fields_out_dev, void* stream);

/* The uniforms b2rl_tree_sample would draw for (seed, rng_offset) in place of torch.multinomial's generator
 * (baseline/PER.py:97) — lets a
 * test replay a device-RNG run through the oracle. */
int b2rl_philox_uniforms(uint64_t seed, uint64_t rng_offset, int64_t n, double* out_dev,
                         void* stream);

/* PER.update (baseline/PER.py:83-90 -> Tree.update :36-42) and
 * PrioritizedMemory.update_priorities (baseline/utils.py:347-350): set
 * priority[idx[k]] = vals[k] for k = 0..n-1 in order — for a duplicated index
 * the LAST occurrence wins — and refresh the touched root paths.
 * Deterministic (no floating-point atomics). */
int b2rl_tree_update(b2rl_replay* h, const int64_t* idx_dev, const float* vals_dev, int64_t n,
                     void* stream);

/* PrioritizedMemory.total_prios (baseline/utils.py:359-360) and
 * PER.max_weight (baseline/PER.py:129-133).  stats_out_dev receives 3
 * doubles: {sum(p), min valid p, max IS weight for `beta`}; max_w_out_dev (may be
 * NULL) receives the max IS weight as one fp32 (the operand of the multi-GPU
 * MAX all-reduce). */
int b2rl_tree_stats(b2rl_replay* h, float beta, double* stats_out_dev, float* max_w_out_dev,
                    void* stream);

/* Tree.prior_torch (baseline/PER.py:17) read-back: priorities of slots
 * [start, start+n) as fp32. */
int b2rl_tree_leaves(b2rl_replay* h, int64_t start, int64_t n, float* out_dev, void* stream);

/* Stored level k of the sum-tree, for tests and diagnostics: the internal node values (Node._reduce,
 * baseline/sumtree.py:21-27) that every draw descends through.  k = 0 fills the shape only: *n_nodes = cap2 (the
 * leaves), *levels = G (stored internal levels), *top_bits = binary levels spanned by the top group.  For k in
 * 1..G, *n_nodes = cap2 >> 4k (1 at k = G, the root), and the nodes' fp64 sums and fp32 minima are copied on
 * `stream` into sums_out_dev / mins_out_dev when those are not null.  levels / top_bits may be NULL.  No kernel. */
int b2rl_tree_level(const b2rl_replay* h, int32_t k, int64_t* n_nodes, int32_t* levels, int32_t* top_bits,
                    double* sums_out_dev, float* mins_out_dev, void* stream);

/* Minibatch assembly of Replay.buffer (APE_X/ReplayMemory.py:61-116,
 * R2D2/ReplayMemory.py:53-122, IMPALA/ReplayMemory.py:30-54): for every
 * field f with out_fields[f] != NULL copy row idx[k] to out_fields[f] + k *
 * field_bytes[f].  Rows that are multiples of 16 B go HBM -> SMEM -> HBM with
 * bulk async copies (TMA); the rest through a vectorised byte kernel. */
int b2rl_replay_gather(b2rl_replay* h, const int64_t* idx_dev, int64_t n,
                       void* const* out_fields_dev, void* stream);

/* Frame-deduplicated Ape-X store.  An Ape-X record (APE_X/Player.py:252-261) carries two frame stacks, s and s', and
 * most of their frames repeat: LocalBuffer.get_traj (APE_X/Player.py:33-57) makes record k's s' record k + 1's s,
 * stacks UNROLL_STEP steps apart share frames, and an episode starts with one frame four times (:203-209).
 *
 * b2rl_dedup_attach turns the replay into one whose field `planes_field` (32 bytes per slot) holds 8 int32 pool ids
 * (planes 0-3 of s, then of s') into a library-owned ring of `pool_frames` 84x84 frames; frame sequence number seq
 * lives in pool slot seq mod pool_frames.  A frame of a pushed batch reuses a stored frame only when that frame has
 * seq >= head - window (head: frames stored before the batch), its key (64-bit content hash & hash_mask) matches and
 * all 7 056 bytes compare equal.  A slot is live while the slot ring has not overwritten it and fewer than
 * pool_frames - window frames have been stored since the batch that inserted it began; slots that stop being live
 * get priority 0 before the pool is overwritten.  hash_mask is for tests (0 makes every frame collide);
 * normal use passes ~0.  Requires window >= 0 and pool_frames - window > 8 (one record) and pool_frames < 2^31.
 *
 * b2rl_dedup_push: PER.push (baseline/PER.py:69-75) of n records on a dedup replay.  s_dev / ns_dev: device (n, 4,
 * 84, 84) uint8 stacks; fields_src: the other fields as for b2rl_replay_push (the planes entry must be NULL).  The
 * call synchronizes `stream` once, to learn how many frames the batch adds.  n <= *max_batch of b2rl_dedup_info.
 * Pushes may come from different streams: each one waits for the previous one's work before it starts.  The host
 * calls themselves must not overlap (one thread at a time, as for every entry point on a handle).
 * b2rl_replay_push, _reserve, _ingest_pipelined, _fill_hash, b2rl_tree_build and b2rl_serve_fill_uniform refuse a
 * dedup replay (b2rl_serve_fill_uniform serves a rollout handle, b2rl_dedup_attach_rollouts below).  b2rl_serve_ring_create / b2rl_serve_fill serve it with the stack store's record layout: the planes
 * field becomes two (B, 4, 84, 84) frame-stack fields (s, then s') in the ring slot, assembled from the pool.
 *
 * b2rl_dedup_info: *pool_dev (the frame pool), *head_seq (frames stored so far), *max_batch (records per push).
 *
 * b2rl_replay_gather_planes: b2rl_replay_gather for a dedup replay, plus the sampled slots' s and s' stacks
 * (Replay.buffer, APE_X/ReplayMemory.py:61-116): stacks_out_dev[0] / [1] (either may be NULL) receive (n, 4, 84,
 * 84) uint8 assembled from planes 0-3 / 4-7 by TMA bulk copies.  out_fields_dev[planes_field] is ignored.
 *
 * The same pool for R2D2 frame strips.  R2D2/Player.py:37-62 (LocalBuffer.get_traj) cuts an episode's sequences with
 * half overlap, so a strip record (b2rl_frames: T + 3 frames, stack t = frames t .. t + 3) shares about half of its
 * frames with the record before it.  b2rl_dedup_attach_strips is b2rl_dedup_attach for records of R =
 * frames_per_record frames each: the planes field holds R int32 pool ids per slot (4 R bytes), frame j of a record
 * having id planes[R slot + j].  Requires pool_frames - window > R; a push takes at most min(capacity, (pool_frames -
 * window - 1) / R, 65536 / R) records.  b2rl_dedup_push_strips is b2rl_dedup_push for it: strips_dev is device
 * (n, R, 84, 84) uint8.  Each push refuses the other kind of handle; b2rl_dedup_info serves both, and so do the
 * refusals above.  b2rl_replay_gather_planes on a strip handle: stacks_out_dev[0] receives the (n, R, 84, 84)
 * strips assembled from the pool and stacks_out_dev[1] must be NULL.  b2rl_serve_ring_create / b2rl_serve_fill
 * serve it with the strip store's record layout: the planes field becomes the (B, R, 84, 84) strip field.
 *
 * The same pool for IMPALA rollouts.  IMPALA/Player.py:88-95 stacks the last four frames, so stack t + 1 repeats three
 * frames of stack t; a rollout's bootstrap stack is the first stack of the same actor's next rollout (:181-203); and
 * checkLength (:116-125) pads a short rollout with the previous rollout's stacks.  A rollout's `state` row (T + 1
 * stacks of 28 224 bytes, IMPALA/ReplayMemory.py:34-43) is R = 4 (T + 1) frames back to back, stack t being frames
 * 4t .. 4t + 3.  b2rl_dedup_attach_rollouts is b2rl_dedup_attach_strips with R = 4 stacks_per_record (T + 1) that
 * also marks the handle as holding rollouts; it takes b2rl_dedup_push_strips with strips_dev the device (n, T + 1,
 * 28 224) uint8 rows, and b2rl_replay_gather_planes / b2rl_serve_fill as for a strip handle (the slot's row is the
 * stack store's `state` row).  Unlike every other dedup replay it is also drawn by b2rl_uniform_fetch (its planes
 * field takes no buffer; the frame rows are those of a stack store, read through plane_stride 4 of b2rl_frames) and
 * b2rl_serve_fill_uniform (the slot's `state` field holds the time-major stacks assembled from the pool, byte for
 * byte the stack store's slot); both require steps + 1 == stacks_per_record.  It has no host-pool form. */
int b2rl_dedup_attach(b2rl_replay* h, int32_t planes_field, int64_t pool_frames, int64_t window, uint64_t hash_mask);
int b2rl_dedup_push(b2rl_replay* h, const uint8_t* s_dev, const uint8_t* ns_dev, const void* const* fields_src,
                    const float* prios, int64_t n, void* stream);
int b2rl_dedup_attach_strips(b2rl_replay* h, int32_t planes_field, int32_t frames_per_record, int64_t pool_frames,
                             int64_t window, uint64_t hash_mask);
int b2rl_dedup_push_strips(b2rl_replay* h, const uint8_t* strips_dev, const void* const* fields_src,
                           const float* prios, int64_t n, void* stream);
int b2rl_dedup_attach_rollouts(b2rl_replay* h, int32_t planes_field, int32_t stacks_per_record, int64_t pool_frames,
                               int64_t window, uint64_t hash_mask);
int b2rl_dedup_info(const b2rl_replay* h, void** pool_dev, int64_t* head_seq, int64_t* max_batch);

/* The strip store of R2D2/ReplayMemory.py:70-88 behind PER.__init__ (baseline/PER.py:49-66), with the frame pool
 * placed where it is read from: b2rl_dedup_attach_strips when pool_on_host is 0; with 1 the pool lives in pinned,
 * mapped host memory owned by the handle (cudaHostAlloc with cudaHostAllocMapped | cudaHostAllocPortable; the kernels
 * address it through cudaHostGetDevicePointer).  The planes field, pool keys, key table, batch scratch and sum-tree
 * stay in device memory.  B2RL_ERR_NOMEM, with the size in the message, when the pinned allocation fails.  A push
 * compares hits and stores misses through the mapped pointer, in order on its stream.  A host pool is never read by
 * bulk async (TMA) copies: b2rl_replay_gather_planes and b2rl_serve_fill copy the sampled slots' strips with 16-byte
 * loads through the mapped pointer, from a few CTAs (B2RL_HOST_GATHER_CTAS, default 8).  b2rl_dedup_info's *pool_dev
 * is then the device alias: never pass it to b2rl_conv1_fused or b2rl_conv1_wgrad.  Ape-X's b2rl_dedup_attach has no
 * placed form.  Arguments are checked before the handle is read. */
int b2rl_dedup_attach_strips_placed(b2rl_replay* h, int32_t planes_field, int32_t frames_per_record,
                                    int64_t pool_frames, int64_t window, uint64_t hash_mask, int32_t pool_on_host);
/* Where the frame pool (the frames of PER.memory, baseline/PER.py:7-28) of a dedup replay lives: *on_host = 1 for
 * pinned host memory, 0 for device; *pool (may be NULL) its host address, or its device address for a device pool. */
int b2rl_dedup_pool_placement(const b2rl_replay* h, int32_t* on_host, void** pool);

/* The strip store with its frames stored encoded, as CompressedDeque.append / __getitem__ (baseline/utils.py:277-296)
 * stores the reference's replay entries, here with a lossless per-frame codec (csrc/frame_codec.cuh, DESIGN.md §4.21):
 * b2rl_dedup_attach_strips whose pool is a ring of P = pool_bytes / 16 units in device memory.  Frame seq's entry
 * seq % pool_frames holds its absolute unit offset and length, so ids, the window and the frame rule are the strip
 * handle's.  A frame takes 1..442 units and never straddles the ring's end (the units skipped count as written).  A hit
 * still needs all 7 056 bytes equal to the stored frame.  A slot also stops being live once P - (window + 1) * 442
 * units or more have been written since its batch began; a push takes at most (P - (window + 2) * 442) / (442 R)
 * records too.  Requires pool_bytes a positive multiple of 16 with P >= 442 (window + 2 + R).  b2rl_replay_gather_planes
 * and b2rl_serve_fill decode the sampled slots' strips (k_decode_planes), byte for byte the strip handle's while the
 * slots are live; a dead or never-written slot decodes to unspecified frames, read inside the pool's allocation (P
 * units plus 7 072 zeroed bytes).  A strip handle's coded pool is never a conv_1 frame source.  Arguments are checked before the handle is read. */
int b2rl_dedup_attach_strips_coded(b2rl_replay* h, int32_t planes_field, int32_t frames_per_record,
                                   int64_t pool_frames, int64_t window, uint64_t hash_mask, int64_t pool_bytes);
/* The Ape-X store (b2rl_dedup_attach, APE_X/ReplayMemory.py:61-116) with its frames stored encoded, the Pairs twin of
 * b2rl_dedup_attach_strips_coded: R = 8, planes 0-3 of s and 4-7 of s'.  Ids, the window, the frame rule, the byte
 * rule and the push bound are those above with R = 8; requires P >= 442 (window + 10).  b2rl_dedup_push stores into
 * it.  b2rl_replay_gather_planes and b2rl_serve_fill decode the sampled slots' s and s' stacks, byte for byte the raw
 * handle's while the slots are live.  Unlike the strip form, conv_1 reads its frames in place: a b2rl_frames source
 * with `offsets` (b2rl_dedup_coded_offsets) decodes each row's four frames on chip.  Arguments are checked before the
 * handle is read. */
int b2rl_dedup_attach_coded(b2rl_replay* h, int32_t planes_field, int64_t pool_frames, int64_t window,
                            uint64_t hash_mask, int64_t pool_bytes);
/* A coded pool's descriptor table, what CompressedDeque (baseline/utils.py:277-296) keeps as its list of pickles:
 * *offsets_dev receives the device int64[pool_frames] absolute unit offsets of the entries (frame id i is encoded at
 * pool + (offsets[i] % P) * 16), the `offsets` of a coded b2rl_frames source. */
int b2rl_dedup_coded_offsets(const b2rl_replay* h, void** offsets_dev);
/* The IMPALA rollout store (b2rl_dedup_attach_rollouts, IMPALA/ReplayMemory.py:14-85) with its frames stored encoded,
 * the rollout twin of b2rl_dedup_attach_strips_coded (DESIGN.md §4.23): R = 4 stacks_per_record, and the handle is
 * marked as holding rollouts.  Ids, the window, the frame rule, the byte rule and the push bound are the strip form's
 * at that R; requires P >= 442 (window + 2 + R).  b2rl_dedup_push_strips stores into it; b2rl_uniform_fetch draws it
 * as the raw rollout store; b2rl_replay_gather_planes decodes the sampled slots' (n, T + 1, 28 224) rows; and
 * b2rl_serve_fill_uniform serves it, decoding the drawn rollouts' stacks time-major after the fill's launch from the
 * slot's idx (a second launch on the same stream), byte for byte the raw rollout store's slot while the slots are
 * live.  Its pool is never a conv_1 frame source: b2rl_dedup_stage_rollouts decodes what a step reads.  Whatever
 * b2rl_dedup_attach_rollouts refuses it refuses with the same message; arguments are checked before the handle. */
int b2rl_dedup_attach_rollouts_coded(b2rl_replay* h, int32_t planes_field, int32_t stacks_per_record,
                                     int64_t pool_frames, int64_t window, uint64_t hash_mask, int64_t pool_bytes);
/* The frames a learner step reads of n drawn rollouts (IMPALA/ReplayMemory.py:30-54, drawn as random.sample draws,
 * baseline/utils.py:310-315) of a coded rollout handle, staged as a small raw frame pool: with R = 4 (T + 1) and
 * idx_dev the device int64[n] slots (b2rl_uniform_fetch's idx, clamped into [0, capacity)), frame c of draw k has pool
 * id planes[R slot + c] % pool_frames; staged_planes_dev[k R + c] (int32[n R]) receives k R + i, i the first of the
 * draw's R positions holding that id, and only those first positions are decoded, into staged_pool_dev + (k R + i)
 * 7 056 (n R frames of 7 056 bytes; the others are left as they were).  conv_1 then reads row k (T + 1) + t of the
 * staged pool through plane_stride 4 of b2rl_frames (pool = staged_pool_dev, planes = staged_planes_dev): stack t of
 * draw k, byte for byte the raw rollout store's while the slot is live.  A dead or never-written slot stages
 * unspecified frames, each read inside the pool's allocation.  One launch, no host synchronisation: capturable in a
 * CUDA graph.  An error, and no launch, unless h is a coded rollout handle, the buffers are non-NULL, staged_pool_dev
 * 16-byte and staged_planes_dev 4-byte aligned, and n R < 2^31. */
int b2rl_dedup_stage_rollouts(b2rl_replay* h, const int64_t* idx_dev, int64_t n, uint8_t* staged_pool_dev,
                              int32_t* staged_planes_dev, void* stream);
/* A coded pool's counters, the sizes CompressedDeque (baseline/utils.py:277-296) leaves to pickle (each may be NULL):
 * units written so far (wrap padding included), P, and frames stored.  Strip, Ape-X and rollout coded handles alike. */
int b2rl_dedup_codec_stats(const b2rl_replay* h, int64_t* units_written, int64_t* pool_units, int64_t* frames_stored);
/* The pool's codec on device buffers, as CompressedDeque.append / __getitem__ (baseline/utils.py:277-296) on one
 * frame: b2rl_frame_encode writes frame j (n frames of 7 056 bytes) to enc_dev + 7 072 j and its length in units to
 * units_dev[j] (units_dev may be NULL); the bytes after the encoding in its 7 072 are left as they were.
 * b2rl_frame_decode is its inverse for encodings at the same stride; any other bytes decode to unspecified frames,
 * each read from its own 7 072 bytes only.  Buffers 16-byte aligned. */
int b2rl_frame_encode(const uint8_t* frames_dev, int64_t n, uint8_t* enc_dev, int32_t* units_dev, void* stream);
int b2rl_frame_decode(const uint8_t* enc_dev, int64_t n, uint8_t* frames_dev, void* stream);
int b2rl_replay_gather_planes(b2rl_replay* h, const int64_t* idx_dev, int64_t n, void* const* stacks_out_dev,
                              void* const* out_fields_dev, void* stream);

/* IMPALA's minibatch for a captured learner step (IMPALA/ReplayMemory.py:30-54, drawn as random.sample draws,
 * baseline/utils.py:310-315) in ONE launch: n rollouts drawn uniformly WITHOUT replacement from the ring's valid
 * region [head - size, head) with exactly the permutation of b2rl_serve_fill_uniform (same slots from the same
 * device-resident Philox state, size and head; the counter advances by n), written into the caller's fixed
 * buffers.  size and head are the host-side values of b2rl_replay_size at the call, so slots reserved by an ingest
 * in flight are never drawn.  idx_out_dev: int64[n].  For each field f with fields_out_dev[f] != NULL (with
 * steps = T): a row of T 4-byte words -> word t of draw k at t * n + k; a 1/2/4/8-byte scalar -> row k.  A frame
 * field (a bulk row of T + 1 equal steps) is not copied and its entry must be NULL: frame_rows_out_dev (int64[(T+1)
 * * n], may be NULL) receives the frame-table rows of the time-major frames instead, row t * n + k = idx[k] * (T+1)
 * + t, for b2rl_conv1_fused / b2rl_conv1_wgrad over the field.  fields_out_dev may be NULL.  An error, and no
 * launch, when n > size, size > 2^32 or a field is not one of those three kinds. */
int b2rl_uniform_fetch(b2rl_replay* h, int64_t n, int32_t steps, int64_t* idx_out_dev,
                       void* const* fields_out_dev, int64_t* frame_rows_out_dev, void* stream);

/* Learner.train target section, Ape-X (APE_X/Learner.py:85-121):
 *   a* = argmax_a qn_online[b,:];  y = r + gamma_n * qn_target[b,a*] * notdone
 *   d = clamp(y - q_s[b,action[b]], -1, 1);  prio = (|d| + 1e-7)^alpha
 *   loss = 0.5 * mean(w * d^2);  grad_q = dLoss/dq_s  (dense B x A)
 * q_* are (B, A) fp32 row-major; action int64[B]; reward/notdone/weight
 * fp32[B].  scalars_out_dev receives 3 floats {loss, mean(y), mean(w)}.
 * Any output pointer may be NULL. */
int b2rl_apex_target(const float* q_s_dev, const float* qn_online_dev, const float* qn_target_dev,
                     const int64_t* action_dev, const float* reward_dev, const float* notdone_dev,
                     const float* weight_dev, int32_t B, int32_t A, float gamma_n, float alpha,
                     float* target_out_dev, float* td_out_dev, float* prio_out_dev,
                     float* grad_q_out_dev, float* scalars_out_dev, void* stream);

/* Learner.train target section, R2D2 (R2D2/Learner.py:110-198) with
 * value_transform / value_inv_transform (:22-35).  Time-major layouts:
 * q, q_target (L, B, A); action int64 (L-1, B); reward fp32 (L-1, B);
 * notdone fp64-valued but passed as fp32[B] (0/1); weight fp32[B].
 * Outputs: target, td (L-1, B); prio fp32[B] =
 * (0.9 max_t|td| + 0.1 mean_t|td|)^alpha; grad_q (L, B, A);
 * scalars {loss, mean q(s,a)}. */
int b2rl_r2d2_target(const float* q_dev, const float* q_target_dev, const int64_t* action_dev,
                     const float* reward_dev, const float* notdone_dev, const float* weight_dev,
                     int32_t L, int32_t B, int32_t A, int32_t n_step, double gamma, float alpha,
                     int32_t use_rescaling, float* target_out_dev, float* td_out_dev,
                     float* prio_out_dev, float* grad_q_out_dev, float* scalars_out_dev,
                     void* stream);

/* V-trace of IMPALA (IMPALA/Learner.py:141-215), (T, B) time-major fp32:
 * pi_a = learner prob of the taken action, mu_a = behaviour prob, value =
 * V(s_t), bootstrap[B] = V(s_T) * done, reward.  Outputs vtarget (T, B)
 * (:202) and advantage (T, B) (:207-212). */
int b2rl_vtrace(const float* pi_a_dev, const float* mu_a_dev, const float* value_dev,
                const float* bootstrap_dev, const float* reward_dev, int32_t T, int32_t B,
                float gamma, float c_lambda, float c_bar, float p_bar, float* vtarget_out_dev,
                float* advantage_out_dev, void* stream);

/* Where conv_1 (b2rl_conv1_fused, b2rl_conv1_wgrad) reads frame row r: a 28 224-byte stack of four 84x84 uint8
 * frames.  Exactly one of three sources is set, the other pointers NULL:
 *   base    row r is at base + r * row_stride (16-byte aligned).  A stride of 28 224 reads whole frame stacks, e.g.
 *           b2rl_replay_field_ptr of the state field.  A stride of 7 056 reads the overlapping 4-frame windows of an
 *           R2D2 frame strip: a sequence of T observations stored as its T + 3 distinct frames, where stack t is
 *           frames t .. t + 3 (R2D2/Player.py:38-63 stacks the last four frames of one episode, and
 *           R2D2/ReplayMemory.py:70-88 stores T such stacks per sequence).
 *   table   ONE device-resident entry (const uint8_t*, 8-byte aligned) that holds `base`, read when the kernels
 *           start, e.g. written by b2rl_serve_bind: a launch captured in a CUDA graph reads whichever served
 *           minibatch slot (Replay_Server.sample, APE_X/ReplayMemory.py:251-257) was bound before the replay.  The
 *           base it holds must be 16-byte aligned.  When b2rl_conv1_wgrad splits a large n over several launches
 *           (idx_dev NULL), each launch adds its row offset to the loaded base on the device.
 *   pool + planes (+ plane_base, plane_stride)   a frame-deduplicated store (b2rl_dedup_attach,
 *           b2rl_dedup_attach_strips): channel c of row r is the 7 056-byte frame pool +
 *           planes[plane_stride r + plane_base + c] * 7 056 (pool 16-byte aligned, planes 4-byte aligned).
 *           plane_stride 0 means 8, the Ape-X layout: plane_base 0 reads `state`, 4 `next_state` of the transition
 *           APE_X/Player.py:252-261 sends.  plane_stride 1 (plane_base 0) reads the overlapping windows of R2D2 strip
 *           records, whose T + 3 pool ids per slot are consecutive: row slot * (T + 3) + t is stack t of the slot.
 *           plane_stride 4 (plane_base 0) reads the stacks of IMPALA rollout records (b2rl_dedup_attach_rollouts),
 *           4 (T + 1) pool ids per slot: row slot * (T + 1) + t is stack t of the slot, as in a stack store.
 *   pool + planes + offsets (+ plane_base, pool_units, pool_frames)   an Ape-X store whose pool is coded
 *           (b2rl_dedup_attach_coded): channel c of row r is the frame encoded at pool + (offsets[id % pool_frames] %
 *           pool_units) * 16, id = planes[8 r + plane_base + c] read as unsigned, decoded on chip into the row's
 *           shared-memory buffer (as CompressedDeque.__getitem__, baseline/utils.py:277-296, decodes an entry before
 *           the learner reads it).  plane_stride must be 0 or 8, pool_units and pool_frames positive, offsets 8-byte
 *           aligned; the pool must have 7 072 readable bytes past its last unit, as a coded handle's has.
 * row_stride (base and table) must be a positive multiple of 16.  Row indices are clamped to [0, rows), rows >= 1:
 * the caller guarantees that row rows - 1 ends inside the allocation.  Zeroed trailing fields (offsets NULL) keep a
 * descriptor's meaning from before they were added. */
typedef struct {
  const uint8_t* base;
  const uint8_t* const* table;
  const uint8_t* pool;
  const int32_t* planes;
  int64_t row_stride;
  int64_t rows;
  int32_t plane_base;
  int32_t plane_stride;
  const int64_t* offsets;
  int64_t pool_units;
  int64_t pool_frames;
} b2rl_frames;

/* Fused gather + first convolution (north-star "TMA staging of sampled transition slices
 * into shared memory for the Q-network's first GEMM"): conv_1 of cfg/ape_x.json / cfg/r2d2.json
 * (8x8, stride 4, 4 -> 32 channels, no bias; baseline/baseNetwork.py:165-172) applied to
 * frames[idx[k]] / 255 (APE_X/Learner.py:61-67,78,85,87) on the Hopper tensor cores (wgmma), for one or
 * two networks (online + target) in one pass; the sampled uint8 frames are never staged in HBM.
 * c_out = 32 (cfg/ape_x.json, cfg/r2d2.json) or 16 (cfg/impala.json:25-37).
 *   b2rl_conv1_pack   w_dev fp32 [c_out][4][8][8] of network `net` -> packed int8 digits
 *                     (bq_out: n_nets*4*c_out*256 bytes) and per-channel scale (scale_out: n_nets*c_out fp32)
 *   b2rl_conv1_fused  frames: the rows' source (host struct), idx_dev int64[n] or NULL (rows 0..n-1), out_dev fp32
 *                     [n_nets][n][20][20][c_out] (NHWC), relu != 0 applies ReLU.  An error, and no launch, for a
 *                     source b2rl_frames does not allow. */
int b2rl_conv1_pack(const float* w_dev, int32_t net, int32_t n_nets, int32_t c_out, int8_t* bq_out_dev,
                    float* scale_out_dev, void* stream);
/* Up to 4 such packs in ONE launch (host arrays of `jobs` entries): the learner step packs the online conv_1 weights
 * for its one-network and its two-network b2rl_conv1_fused launch and the target weights for the latter
 * (APE_X/Learner.py:78,85,87 evaluate conv_1 with both parameter sets every step). */
int b2rl_conv1_pack_jobs(const float* const* w_dev, const int32_t* net, const int32_t* n_nets,
                         int8_t* const* bq_out_dev, float* const* scale_out_dev, int32_t jobs, int32_t c_out,
                         void* stream);
int b2rl_conv1_fused(const b2rl_frames* frames, const int64_t* idx_dev, int64_t n, const int8_t* bq_dev,
                     const float* scale_dev, int32_t n_nets, int32_t c_out, float* out_dev, int32_t relu,
                     void* stream);

/* Weight gradient of conv_1 fused with the gather (the backward half of b2rl_conv1_fused;
 * loss.backward() in APE_X/Learner.py:123-138 for baseline/baseNetwork.py:165-172's first layer):
 *   gw[co][c][ky][kx] (+)= (1/255) * sum_{k,oy,ox} gy[k][oy][ox][co] * frames[idx[k]][c][4oy+ky][4ox+kx]
 * frames: as for b2rl_conv1_fused; gy_dev: [n][20][20][c_out] fp32 (NHWC); y_relu_dev: NULL, or the post-ReLU output
 * of b2rl_conv1_fused(relu = 1) for the same rows — gy is then the gradient w.r.t. that output and is masked by
 * (y > 0) on the fly (the ReLU's backward); gw_dev: [c_out][4][8][8] fp32; workspace_dev:
 * b2rl_conv1_wgrad_workspace_floats(c_out) floats of scratch (per-SM partial sums, summed in fp64 in a
 * fixed order: the result is deterministic).  idx_dev may be NULL (rows 0..n-1). */
int64_t b2rl_conv1_wgrad_workspace_floats(int32_t c_out);
int b2rl_conv1_wgrad(const b2rl_frames* frames, const int64_t* idx_dev, int64_t n, const float* gy_dev,
                     const float* y_relu_dev, int32_t c_out, float* workspace_dev, float* gw_dev, int32_t accumulate,
                     void* stream);

/* The stem of the IMPALA residual network (netCat RESCNN2D, Espeholt et al. 2018 Fig. 3): a 3x3 / stride-1 / pad-1,
 * 4 -> 16 channel bias-free conv of frames[idx[k]] / 255 followed by a 3x3 / stride-2 / pad-1 max-pool, fused with
 * the gather (the RESCONV2D node of baseline/baseNetwork.py:796-820 cannot be built, and describes a different
 * block; the convs are bias-free as its conv2D helper's, baseline/baseNetwork.py:742-760); the frames are read as
 * conv_1 reads them, from any b2rl_frames source except a coded pool and
 * plane_stride 0 / 8 (Ape-X's transition pairs).  Deterministic: no atomics, fixed summation orders.
 *   b2rl_stem_pack   w_dev fp32 [16][4][3][3] -> packed int8 digits (bq_out: 3 072 bytes, 16-byte aligned) and
 *                    per-channel scale (scale_out: 16 fp32)
 *   b2rl_stem_fused  pooled_out_dev fp32 [n][16][42][42] (NCHW), argmax_out_dev uint8 [n][16][42][42]: 3i + j of
 *                    the window position (row 2py - 1 + i, column 2px - 1 + j) that holds the first maximum in
 *                    row-major window order, padded positions never chosen (torch's max_pool2d picks the same one)
 *   b2rl_stem_fused_pair  b2rl_stem_fused of two networks over the same rows in one launch (R2D2's online and target
 *                    nets, the burn-in and window forwards of R2D2/Learner.py:99-104,121,132): each stack is loaded
 *                    and zero-bordered once and run against both packs.  bq_dev: the two nets' packs, 3 072 bytes
 *                    each, back to back (16-byte aligned); scale_dev: 2 x 16 fp32; pooled_out_dev fp32
 *                    [2][n][16][42][42] (net 0's n stacks, then net 1's); argmax_out_dev uint8 [n][16][42][42], net
 *                    0's argmax, or NULL for none.  Each net's pooled output (and net 0's argmax) is bit for bit what
 *                    b2rl_stem_fused writes with that net's pack.
 *   b2rl_stem_wgrad  gw[co][c][ky][kx] (+)= dL/dW from the same rows, the pooled gradient gpooled_dev fp32
 *                    [n][16][42][42] and the forward's argmax (16-byte aligned); workspace_dev:
 *                    b2rl_stem_wgrad_workspace_doubles() doubles of per-SM partial sums. */
int b2rl_stem_pack(const float* w_dev, int8_t* bq_out_dev, float* scale_out_dev, void* stream);
int b2rl_stem_fused(const b2rl_frames* frames, const int64_t* idx_dev, int64_t n, const int8_t* bq_dev,
                    const float* scale_dev, float* pooled_out_dev, uint8_t* argmax_out_dev, void* stream);
int b2rl_stem_fused_pair(const b2rl_frames* frames, const int64_t* idx_dev, int64_t n, const int8_t* bq_dev,
                         const float* scale_dev, float* pooled_out_dev, uint8_t* argmax_out_dev, void* stream);
int64_t b2rl_stem_wgrad_workspace_doubles(void);
int b2rl_stem_wgrad(const b2rl_frames* frames, const int64_t* idx_dev, int64_t n, const float* gpooled_dev,
                    const uint8_t* argmax_dev, double* workspace_dev, float* gw_dev, int32_t accumulate, void* stream);

/* Learner.step (APE_X/Learner.py:123-138; IMPALA/Learner.py:258-266 without the clipping) with
 * torch.optim.RMSprop's update (baseline/utils.py getOptim :124-130; centered for Ape-X,
 * cfg/ape_x.json:27-35) in ONE pass: square_avg / grad_avg / param update, gradient zeroed, and
 * the reference's diagnostic "norm" sqrt(sum_i ||g_i||_2) written to grad_norm_out_dev (may be
 * NULL).  The four pointer arrays and numel are HOST arrays of n_tensors (<= 24) entries holding
 * device pointers of dense tensors with identical element order; sumsq_scratch_dev: n_tensors
 * doubles, zeroed once by the caller (the kernel re-zeroes them).  images (may be NULL): a HOST array of
 * 6 * n_tensors int64 {fwd image, W^T image, rows, cols, total_n, n_off}; a tensor whose image pointers are not both
 * 0 is a row-major rows x cols weight (multiples of 32) of a stack of total_n rows (the sibling heads of
 * cfg/ape_x.json:52-71) at row n_off, and the update also writes it into the stack's 3xTF32 B-role images
 * (b2rl_gemm_split_pack_into with total_rows = total_n, total_k = cols; and its transpose, total_rows = cols,
 * total_k = total_n), bit-equal to packing the updated weights. */
int b2rl_rmsprop_step(float* const* params, float* const* grads, float* const* square_avg,
                      float* const* grad_avg, const int64_t* numel, int32_t n_tensors, double lr, double alpha,
                      double eps, int32_t centered, const int64_t* images, double* sumsq_scratch_dev,
                      float* grad_norm_out_dev, void* stream);
/* The same update issued in two parts: Learner.step (APE_X/Learner.py:123-138) has no gradient clipping, so a
 * parameter can be updated as soon as its own gradient is final — the dense heads' (97 % of the elements) while the
 * convolution stack's backward still runs.  Each part calls b2rl_rmsprop_step on its tensors with
 * grad_norm_out_dev = NULL and sumsq_scratch_dev pointing at its slots of one n-entry scratch; this call then forms
 * the reference's "norm" sqrt(sum_i ||g_i||_2) (:130) over all n slots and re-zeroes them. */
int b2rl_rmsprop_norm_finish(double* sumsq_scratch_dev, int32_t n_tensors, float* grad_norm_out_dev, void* stream);

/* The dense heads of the networks (nn.Linear, bias-free: baseline/baseNetwork.py:77-79; 3136 -> 512
 * adv/val heads cfg/ape_x.json:52-71) at fp32 accuracy on the tensor cores: every fp32 operand is
 * split into two TF32 terms and C (+)= A[M][K] * B[N][K]^T is formed from three wgmma products
 * with fp32 accumulation.  `split_pack` turns a row-major fp32 matrix (or its transpose) into the
 * operand image (b_role = 0: the A / M side, 1: the B / N side); `packed_floats` is the size of
 * that image in floats.  Shapes with few output tiles split K over the SMs; their partial tiles go to
 * workspace_dev (b2rl_gemm_workspace_floats floats, 0 = not needed) and are summed in a fixed order,
 * so the result is deterministic. */
int64_t b2rl_gemm_packed_floats(int64_t rows, int64_t k, int32_t b_role);
int b2rl_gemm_split_pack(const float* src_dev, int64_t src_rows, int64_t src_cols, int64_t src_ld,
                         int32_t transpose, int32_t b_role, float* out_dev, void* stream);
/* One piece of an operand (stacked weight matrices of sibling heads, cfg/ape_x.json:52-71): image rows [row_offset, +rows), contraction
 * [k_offset, +k) of a total_rows x total_k operand; offsets (and inner piece sizes) multiples of 32. */
int b2rl_gemm_split_pack_into(const float* src_dev, int64_t src_rows, int64_t src_cols, int64_t src_ld,
                              int32_t transpose, int32_t b_role, float* out_dev, int64_t total_rows,
                              int64_t total_k, int64_t row_offset, int64_t k_offset, void* stream);
/* The two element-wise steps between the conv stack and the heads — the act_3 ReLU and nn.Flatten of
 * cfg/ape_x.json:37-51 (baseline/baseNetwork.py:204-209) — folded into the heads' operand packing.  y_dev is the conv
 * stack's output as it lies in memory (NHWC: [B][HW][C]); the images index features in the NCHW-flatten order
 * f = c*HW + hw the reference's weights use.  transpose = 0: A-role image of x = relu(y) as [B][C*HW] (forward);
 * transpose = 1: B-role image of x^T (the heads' weight gradient).  b2rl_unflatten_relu_mask is their backward:
 * out[b][hw][c] = gx[b][c*HW + hw] * (y[b][hw][c] > 0). */
int b2rl_gemm_pack_act_nhwc(const float* y_dev, int64_t B, int64_t HW, int64_t C, int32_t relu, int32_t transpose,
                            float* out_dev, void* stream);
int b2rl_unflatten_relu_mask(const float* gx_dev, int64_t gx_ld, int32_t splits, int64_t split_stride,
                             const float* y_dev, int64_t B, int64_t HW, int64_t C, float* out_dev, void* stream);
int64_t b2rl_gemm_workspace_floats(int64_t M, int64_t N, int64_t K, int64_t ldc);
int b2rl_gemm_tf32x3(const float* a_packed_dev, const float* b_packed_dev, float* c_dev, int64_t M,
                     int64_t N, int64_t K, int64_t ldc, float* workspace_dev, void* stream);
/* The heads' GEMM (nn.Linear, baseline/baseNetwork.py:77-79) without its split-K reduction: the `splits` partials
 * (splits = b2rl_gemm_workspace_floats / (M * ldc), or 1 when that is 0) are stored as [split][M][ldc] at
 * partials_dev, which holds max(b2rl_gemm_workspace_floats, M * ldc) floats.  Their consumer sums them in split
 * order, which gives the bits b2rl_gemm_tf32x3 returns: b2rl_dueling_forward and b2rl_unflatten_relu_mask take
 * (splits, split_stride = M * ldc) for that. */
int b2rl_gemm_tf32x3_partials(const float* a_packed_dev, const float* b_packed_dev, float* partials_dev, int64_t M,
                              int64_t N, int64_t K, int64_t ldc, void* stream);

/* Tail of the dueling Q-network after the first dense layer of the two heads (cfg/ape_x.json:52-88: MLP
 * heads 3136-512-A and 3136-512-1, then the Add / Mean / Substract nodes executed by
 * baseline/baseAgent.py:287-309):  r = relu(h);  Q_j = r[:H].Wa[j] + r[H:].Wv - mean_i(r[:H].Wa[i]).
 * h_dev: [M][2H] pre-activations (advantage | value), wa_dev: [A][H], wv_dev: [H], q_dev: [M][A].
 * backward: gh_dev [M][2H] (may be NULL), gwa_dev [A][H] and gwv_dev [H] (both or neither), row_ws_dev:
 * M*(A+1) floats of scratch; sums over the batch run in a fixed order.  H % 32 == 0, H <= 1024, A <= 32.
 * forward: h_dev holds `splits` partials of h, split_stride floats apart (b2rl_gemm_tf32x3_partials; 1 and 0 for a
 * plain h), summed in split order; h_out_dev (may be NULL) receives the summed h.  h_dev, h_out_dev 16-byte aligned. */
int b2rl_dueling_forward(const float* h_dev, int32_t splits, int64_t split_stride, int64_t M, int64_t H,
                         const float* wa_dev, int64_t A, const float* wv_dev, float* q_dev, float* h_out_dev,
                         void* stream);
int b2rl_dueling_backward(const float* h_dev, const float* gq_dev, int64_t M, int64_t H, const float* wa_dev,
                          int64_t A, const float* wv_dev, float* gh_dev, float* gwa_dev, float* gwv_dev,
                          float* row_ws_dev, void* stream);
/* The weight-gradient half alone (dL/dW of the heads' second layers, cfg/ape_x.json:52-71; part of loss.backward(),
 * APE_X/Learner.py:123-138), from the row table a previous b2rl_dueling_backward (with gwa_dev = NULL)
 * left in row_ws_dev: lets the caller run it on another stream than the dL/dh half. */
int b2rl_dueling_backward_w(const float* h_dev, const float* row_ws_dev, int64_t M, int64_t H, int64_t A,
                            float* gwa_dev, float* gwv_dev, void* stream);

/* Device serve ring: the stand-alone replay server's minibatch transport without the host
 * (APE_X/ReplayServer.py:41-114 serves pickled minibatches over the Redis list `BATCH` and applies the
 * pickled `update` list; APE_X/ReplayMemory.py:170-257 is the learner-side consumer).  ONE cudaMalloc
 * allocation owned by the server process holds `slots` minibatch slots followed by `slots` update slots:
 *   minibatch slot: header {uint64 seq, int64 n} | idx int64[B] | w fp32[B] | field f: B rows of
 *                   field_bytes[f] (the replay's fields in order)
 *   update slot:    header {uint64 seq, int64 n} | idx int64[B] | prio fp32[B]
 * Every array starts on a 16-byte boundary, every slot on a 128-byte boundary.  The learner process maps the
 * allocation through CUDA IPC (on the same GPU or a peer GPU); the handshake that orders the two processes'
 * streams is host-level (Redis descriptors + interprocess CUDA events): nothing on the device waits for the
 * other process. */
#define B2RL_IPC_HANDLE_BYTES 64
typedef struct b2rl_serve_ring b2rl_serve_ring; /* opaque */
typedef struct {
  int64_t batch;                          /* B: transitions per minibatch slot          */
  int64_t slots;                          /* K: minibatch slots (and as many update slots) */
  int64_t n_fields;
  int64_t field_bytes[B2RL_MAX_FIELDS];
  int64_t field_off[B2RL_MAX_FIELDS];     /* field f's B rows inside a minibatch slot   */
  int64_t idx_off, w_off;                 /* inside a minibatch slot (header at 0)      */
  int64_t slot_bytes;                     /* stride of the minibatch slots              */
  int64_t upd_idx_off, upd_prio_off;      /* inside an update slot (header at 0)        */
  int64_t upd_slot_bytes;                 /* stride of the update slots                 */
  int64_t upd_base;                       /* offset of update slot 0 (= slots * slot_bytes) */
  int64_t total_bytes;
} b2rl_serve_layout;

/* The layout of a ring for a replay with these fields (host arithmetic only, no CUDA call): the slot geometry
 * the ReplayServer's `BATCH` blobs carry, APE_X/ReplayServer.py:65-114. */
int b2rl_serve_layout_init(int64_t batch, int32_t slots, int32_t n_fields, const int64_t* field_bytes,
                           b2rl_serve_layout* out);
/* ReplayServer.__init__ (APE_X/ReplayServer.py:20-39, R2D2/ReplayServer.py:20-39): allocate the ring for replay
 * `h` on h's device (headers zeroed).  Any field with row_bytes >= 1 can be served. */
int b2rl_serve_ring_create(b2rl_replay* h, int64_t batch, int32_t slots, b2rl_serve_ring** out);
/* The ring's layout (what a learner needs besides the IPC handle to open it; APE_X/ReplayMemory.py:170-186). */
int b2rl_serve_ring_layout(const b2rl_serve_ring* r, b2rl_serve_layout* out);
/* cudaIpcGetMemHandle of the ring's allocation: B2RL_IPC_HANDLE_BYTES bytes to handle_out (stands in for the
 * Redis connection the consumer opens, APE_X/ReplayMemory.py:170-186). */
int b2rl_serve_ring_export(const b2rl_serve_ring* r, void* handle_out);
/* Replay_Server.__init__ (APE_X/ReplayMemory.py:170-186), learner side: map an exported ring into this process
 * on `device` (cudaIpcOpenMemHandle with lazy peer access: the server may sit on another GPU).  `layout` must be
 * the server's; it is checked against the arithmetic of b2rl_serve_layout_init.  Release with
 * b2rl_serve_ring_close; a ring made by b2rl_serve_ring_create is released with b2rl_serve_ring_destroy. */
int b2rl_serve_ring_open(const void* handle, const b2rl_serve_layout* layout, int32_t device, b2rl_serve_ring** out);
int b2rl_serve_ring_close(b2rl_serve_ring* r);
int b2rl_serve_ring_destroy(b2rl_serve_ring* r);
/* Device pointers of slot k's arrays (the members of one `BATCH` blob, APE_X/ReplayServer.py:95-114, and of one
 * `update` entry, :41-63), valid in this process: batch_out[0..2+n_fields] = {header, idx, w, field 0, ...},
 * update_out[0..2] = {header, idx, prio}.  Either may be NULL. */
int b2rl_serve_slot_ptrs(const b2rl_serve_ring* r, int32_t slot, void** batch_out, void** update_out);
/* ReplayServer.buffer (APE_X/ReplayServer.py:65-114, R2D2/ReplayServer.py:65-136) for one minibatch, in ONE
 * launch: B draws from h's device-resident Philox stream with the descent and IS-weight arithmetic of
 * b2rl_tree_sample_fetch (the counter advances by B), idx / w / 1-2-4-8-byte scalar fields written by the drawing
 * threads, bulk rows (a multiple of 16 bytes, >= 1024) copied HBM -> SMEM -> slot with TMA bulk copies as
 * b2rl_replay_gather does, every other row (e.g. R2D2's 80-step action / reward) copied in words or bytes by the
 * other threads of the same CTAs, and the header {seq, B} written last.  The CTAs split the minibatch's copy work
 * evenly, so a minibatch of fewer draws than SMs still uses every SM.  The slot equals b2rl_tree_sample_fetch +
 * b2rl_replay_gather from the same RNG state, bit for bit.  max_w_dev: as for b2rl_tree_sample. */
int b2rl_serve_fill(b2rl_replay* h, b2rl_serve_ring* r, int32_t slot, uint64_t seq, float beta,
                    const float* max_w_dev, void* stream);
/* IMPALA's minibatch (IMPALA/ReplayMemory.py:30-54: s[T+1, B], a[T, B], mu[T, B], r[T, B], done[B]) in ONE launch:
 * B rollouts drawn uniformly WITHOUT replacement from the ring's valid region [head - size, head), as random.sample
 * draws them (baseline/utils.py:310-315), written TIME-MAJOR into minibatch slot `slot`.  Draw k is slot
 * (tail + pi(k)) mod capacity, tail = (head - size) mod capacity, where pi is a permutation of [0, size): a 4-round
 * balanced Feistel network on the smallest even bit width >= 2 covering size, cycle-walked into [0, size), with the
 * four words of the Philox4x32-10 block of the handle's device-resident stream at its current counter as round keys
 * (the counter advances by B).  size and head are the host-side values of b2rl_replay_size at the call.  Field
 * layout, with steps = T: a bulk row of (T + 1) equal steps -> step t of draw k at row t * B + k; a row of T 4-byte
 * words -> word t of draw k at t * B + k; a 1/2/4/8-byte scalar -> row k.  idx is written, w is not (uniform replay
 * has no IS weights), the header {seq, B} last.  Same slot layout and ring as b2rl_serve_fill.  An error, and no
 * launch, when B > size or the ring was not created for h.  Of the frame-deduplicated replays it serves the rollout
 * handle (b2rl_dedup_attach_rollouts) only, assembling each drawn rollout's T + 1 stacks from the frame pool in the
 * same launch; a coded rollout handle's stacks are decoded by a second launch (b2rl_dedup_attach_rollouts_coded). */
int b2rl_serve_fill_uniform(b2rl_replay* h, b2rl_serve_ring* r, int32_t slot, uint64_t seq, int32_t steps,
                            void* stream);
/* Replay_Server.sample (APE_X/ReplayMemory.py:251-257) without the unpickle: copy minibatch slot k (slot_bytes,
 * header included) to dst_dev with one cudaMemcpyAsync on `stream` (a peer copy when the ring is on another GPU). */
int b2rl_serve_take(const b2rl_serve_ring* r, int32_t slot, void* dst_dev, void* stream);
/* Replay_Server.sample (APE_X/ReplayMemory.py:251-257) for a captured learner step (APE_X/Learner.py:55-121), in
 * ONE launch on `stream`: the filled minibatch slot at slot_dev (a mapped ring slot, or a learner-local copy made
 * with b2rl_serve_take), laid out by `layout`, is bound to the step's fixed buffers.  The header {seq, n}, idx and
 * w are copied to header_out_dev (16 B), idx_out_dev (int64[n]) and w_out_dev (fp32[n]).  For each field f:
 * fields_out_dev[f] != NULL receives a copy of its n rows; table_out_dev[f] != NULL (an 8-byte aligned device
 * entry, the `table` of a b2rl_frames source) receives the device address of its rows instead, so
 * the frames are read in the slot.  Either host array may be NULL.  An error, and no launch, for a null slot, a slot
 * base that is not 16-byte aligned or a layout whose batch is not n.  The slot must stay unreleased until the last
 * kernel that reads a table entry has run. */
int b2rl_serve_bind(const void* slot_dev, const b2rl_serve_layout* layout, int64_t n, uint64_t* header_out_dev,
                    int64_t* idx_out_dev, float* w_out_dev, void* const* fields_out_dev, void* const* table_out_dev,
                    void* stream);
/* Replay_Server.update (APE_X/ReplayMemory.py:188-190, flushed to `update` at :241-249): write n <= B (idx,
 * priority) pairs and the header {seq, n} into update slot j, one launch on `stream`. */
int b2rl_serve_put_update(b2rl_serve_ring* r, int32_t slot, uint64_t seq, const int64_t* idx_dev,
                          const float* prio_dev, int64_t n, void* stream);

/* The actors' pickled records decoded on the device (DESIGN.md §4.24), in place of the learner's pickle.loads of each
 * record (APE_X/ReplayMemory.py:74, R2D2/ReplayMemory.py:63) and the host decoders after it.  n records of one template are staged at
 * `stride` bytes apart in blobs_dev (16-byte aligned; stride a multiple of 16 and at least tmpl_len + 16, the last
 * 16 bytes readable), record r being lengths_dev[r] bytes long.  The template: its tmpl_len bytes at tmpl_dev and
 * n_runs runs of 8 int32 at runs_dev ([op, src, len, field, dst, count, aux, kinds], wire.py), dealt to CTAs by the
 * n_tasks [begin, end) run ranges at tasks_dev.  Record r compares its skeleton runs with the template's bytes and
 * writes its values into row rows_dev[r] (r when rows_dev is NULL) of each field: fields_dev[f] (a host array of
 * n_fields device pointers) with row_bytes[f] bytes per row.  status_dev (int32[n_rows], zeroed by the caller, so that
 * several templates can decode into one batch) has ORed into the record's row 1 (skeleton mismatch, the length
 * included), 2 (a value out of range of its field) or 4 (an R2D2 stack that is not the previous one shifted by one
 * frame): it stays 0 for a record decoded.  A row whose status is not 0 holds undefined values.  One launch on
 * `stream`; arguments are checked before it. */
int b2rl_wire_decode(const uint8_t* blobs_dev, int64_t stride, const int32_t* lengths_dev, int64_t n,
                     const uint8_t* tmpl_dev, int32_t tmpl_len, const int32_t* runs_dev, int32_t n_runs,
                     const int32_t* tasks_dev, int32_t n_tasks, const int32_t* rows_dev, void* const* fields_dev,
                     const int64_t* row_bytes, int32_t n_fields, int32_t* status_dev, int64_t n_rows, void* stream);
/* Host side of the same ingest (APE_X/ReplayMemory.py:74, R2D2/ReplayMemory.py:63): blob i (src[i], lengths[i] <= stride bytes) -> dst + i * stride, and its length ->
 * lengths_out[i] (int32).  A plain memcpy loop, so a caller through ctypes holds no interpreter lock meanwhile. */
int b2rl_wire_gather(const void* const* src, const int64_t* lengths, int64_t n, uint8_t* dst, int64_t stride,
                     int32_t* lengths_out);

/* Number of kernels this library has launched in this process (bench.py's
 * `gpu_launches`). */
int64_t b2rl_launch_count(void);

/* Replay-sharded data parallelism (SURVEY.md §8e; the reference has one learner process and no collective:
 * APE_X/Learner.py:123-138 steps a single model).  Mean all-reduce of the SMALL gradient slice that is left when
 * backward ends (the convolution stack: 0.3 MB) across the learner ranks of one node, as one kernel per rank over
 * NVLink / NVSwitch peer memory: stage -> per-CTA flag to every peer -> read every rank's staged slice through the
 * peer mapping, add in rank order (bit-identical on all ranks), scale, write data_dev in place.
 * stage_ptrs_dev / flag_ptrs_dev: DEVICE arrays of `world` device pointers — rank r's staging buffer
 * (2 * stage_cap_floats floats) and flag pad (world * b2rl_peer_allreduce_max_ctas() uint32, zeroed once), both
 * mapped into this process (CUDA IPC / VMM; the Python host uses torch symmetric memory).  epoch_dev:
 * max_ctas uint32 zeroed once, private to the rank; error_dev: set to 1 if a peer never arrived (bounded spin).
 * Every rank must call it the same number of times with the same n. */
int32_t b2rl_peer_allreduce_max_ctas(void);
int b2rl_peer_allreduce_mean(const uint64_t* stage_ptrs_dev, const uint64_t* flag_ptrs_dev, int32_t rank,
                             int32_t world, int64_t stage_cap_floats, float* data_dev, int64_t n,
                             uint32_t* epoch_dev, uint32_t* error_dev, void* stream);
/* The LARGE slice (the dense heads' 12.9 MB, cfg/ape_x.json:52-71) as reduce-scatter + all-gather in one kernel:
 * the gradient bucket itself is peer-mapped (bucket_ptrs_dev[r] = rank r's slice start, n floats); rank r reduces
 * floats [r * slice_floats, ...) of every rank's bucket in rank order into its own bucket and into its result buffer
 * (result_ptrs_dev[r]: 2 * slice_floats floats), then gathers every peer's result.  Flag pads: 2 * world * max_ctas
 * uint32 per rank, zeroed once.  `ctas` CTAs (<= max_ctas, the same on every rank); launched on the stream that
 * produced the gradients, it overlaps the rest of backward (SURVEY.md §8e: new work, no reference counterpart). */
int b2rl_peer_allreduce_mean_big(const uint64_t* bucket_ptrs_dev, const uint64_t* result_ptrs_dev,
                                 const uint64_t* flag_ptrs_dev, int32_t rank, int32_t world, int64_t n,
                                 int64_t slice_floats, int32_t ctas, uint32_t* epoch_dev, uint32_t* error_dev,
                                 void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2RL_H_ */
