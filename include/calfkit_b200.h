/* calfkit_b200.h — C-ABI of libcalfkit_b200.so (sm_90a, H100).
 *
 * The reference (calf-ai/calfkit-sdk v0.2.5) has no FFI for this path: its per-record hot loop is
 *   FastStream decoder -> Envelope validation      calfkit/nodes/base.py:151, calfkit/models/envelope.py:9-17
 *   BaseNodeDef.handler / prepare_context           calfkit/nodes/base.py:64-68,149-164
 *   ToolNodeDef.run                                  calfkit/nodes/tool.py:37-86
 *   BaseNodeDef._publish_action -> broker.publish    calfkit/nodes/base.py:70-147
 *   handler return -> publisher(publish_topic)       calfkit/worker/worker.py:52-53
 * The entry points below are what a ctypes binding underneath calfkit.worker.Worker would bind to
 * replace that loop batch-wise (binding shown in INTEGRATION.md).  Plain C: int status (0 = ok),
 * caller-owned buffers, no exceptions, no torch types.  A bad record never fails a batch: per-record
 * status codes live in the column table (ck_common.h).
 *
 * Threading: one handle = one CUDA stream; calls on one handle must be serialised by the caller,
 * different handles are independent (use two for double buffering).  Calls that launch work return
 * once it is enqueued; ck_sync / ck_fetch_* wait for it.
 */
#ifndef CALFKIT_B200_H
#define CALFKIT_B200_H

#include <stdint.h>
#include "../calfkit-sdk_b200/csrc/ck_common.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ck_handle ck_handle;

typedef struct {           /* one publish; mirrors struct ck_pub in csrc/ck_kernels.cuh */
    uint32_t payload;      /* index into the payload offsets, 0xffffffff = slot unused */
    int32_t  topic_id;     /* registered topic id, or -1: read the name at (record, topic_off, topic_len) */
    uint32_t topic_off, topic_len;
    uint32_t record;       /* input record this publish derives from */
    uint32_t has_key;      /* 1: key = correlation id bytes (nodes/base.py:86,103,117,134) */
    int32_t  partition;    /* murmur2(key) % num_partitions, -1 when unkeyed */
    uint32_t pad;          /* FNV-1a of the topic name (set when the name was looked up): groups unregistered topics */
} ck_publish;

typedef struct {           /* one frame of a frame pass; mirrors struct ck_frame_ent in csrc/ck_kafka.cuh */
    int32_t  topic_id;     /* registered topic id */
    int32_t  partition;    /* -1: unkeyed records (the handler-return publish, worker/worker.py:52-53): the producer picks;
                              with a sticky partition set for the topic (ck_set_sticky_partitions) they are in that one */
    uint32_t n_records;
    uint32_t first;        /* first record, counted in group order */
    int64_t  offset;       /* into the frame bytes */
    int64_t  length;       /* 12 + batchLength */
} ck_frame;

/* lifecycle ------------------------------------------------------------------------------------ */
int  ck_create(int device, uint64_t max_in_bytes, uint64_t max_out_bytes, uint32_t max_records,
               uint32_t max_payloads /* >= max_records; fan-out needs records * (fanout + 1) */,
               uint64_t max_aux_bytes, ck_handle** out);
void ck_destroy(ck_handle* h);
const char* ck_last_error(ck_handle* h);          /* h may be NULL: error of the last failed ck_create */
int  ck_version(void);

/* routing table: replaces the implicit "one FastStream subscriber per node.subscribe_topics"
 * binding of Worker.register_handlers (calfkit/worker/worker.py:33-55).  names = concatenated UTF-8
 * topic strings, offsets[n+1]; ids = caller-chosen non-negative ids. Re-registering replaces. */
int  ck_register_topics(ck_handle* h, const uint8_t* names, const uint32_t* offsets, uint32_t n,
                        const int32_t* ids, uint32_t num_partitions);

/* configure the handle for one @agent_tool node (calfkit/nodes/tool.py:24-35,89-95).
 * publish_topic_id: registered id of node.publish_topic or -1.
 * Result template (optional, nparts > 0): the tool's return value is the JSON string made of
 * literal pieces (kind 0, already JSON-escaped) and raw string arguments (kind 1, blob = key name),
 * at most 5 parts (more is an error: the splice would not fit one output descriptor);
 * nparts == 0: results are supplied by the host through ck_tool_plan(aux). */
int  ck_set_tool_node(ck_handle* h, int32_t publish_topic_id, uint32_t nparts, const uint32_t* kinds,
                      const uint8_t* blob, const uint32_t* part_offsets);

/* decode: copy a batch of records (concatenated bytes + n+1 offsets, pinned or pageable host
 * memory) to HBM and run validate+extract: records in the canonical spelling (what the reference's
 * model_dump_json() emits) are recognised in place; any other valid spelling is re-emitted canonically
 * on the device first (ck_fetch_overlay returns those bytes); invalid ones get a per-record status.
 * ck_submit_device: the batch is already resident (device pointers stay owned by the caller and must
 * outlive the following plan/emit calls; at least 64 readable bytes must follow the last record:
 * the kernels read whole aligned vectors). */
int  ck_submit(ck_handle* h, const uint8_t* host_in, const int64_t* host_off, uint32_t n);
int  ck_submit_device(ck_handle* h, const uint8_t* dev_in, const int64_t* dev_off, uint32_t n);

/* engine options.  option 1 (bucket): value != 0 -> every submitted batch is bucketed by record length (stable radix sort of
 * the record indices on the device) before the thread-per-record walk, so that the lanes of a warp walk records of one size
 * class; for topics with mixed sizes / shapes (reference analogue: none — the reference handles one record at a time).
 * option 2 (frame_bytes): the window W of the frame split of ck_encode_frames; a frame holds at most 61 + W + one record
 * bytes (default 1 MiB)
 * option 3 (frame codec): Kafka's compression codec id of the frames ck_encode_frames, ck_encode_frames_records and
 * ck_encode_recordbatch build: 0 = none (default), 3 = LZ4; any other value is refused.  With LZ4 every frame is a batch with
 * attributes 3 whose records section is one LZ4 frame (descriptor 04224D18 60 40 82: independent 64 KB blocks, no
 * checksums), compressed on the device; a block that would not shrink is stored raw.  The split rule and the frame table
 * keep their meaning (W applies to the uncompressed records); ck_frames_size, ck_fetch_frames_async and the frame table
 * report the compressed frames, each at most its uncompressed length + 4 bytes per 64 KB block + 11
 * option 4 (compression level, Kafka's compression.lz4.level): the LZ4 parse of the following passes.  0 (default), 1 and 2:
 * the greedy parse; 3 .. 17: a hash-chain search of 4 candidates per position at level 3, doubling per level up to 256 at
 * level 9 and above, with a lazy step.  Any other value is refused.  It applies to LZ4 passes only; the frame format, and
 * output that is byte-identical at 0, 1 and 2, do not change.  A pass keeps the level it was queued with (a rewrite into
 * grown buffers uses it again) */
int  ck_set_option(ck_handle* h, uint32_t option, uint64_t value);

/* group the publish table of the current plan by destination topic on the device (stable two-pass radix sort over 12-bit
 * keys: 0 = topic without a registered id, 1 + id = registered topic, 4095 = unused slot) — the per-topic split a producer
 * needs (reference: one broker.publish per topic, nodes/base.py:82-87) without any host-side scan of the table.
 * ck_fetch_groups: order[n_publishes] = publish indices grouped by key (send order kept inside a group) and
 * key_counts[4096]; wait = 0 queues the copies only (page-locked destinations, ck_sync before reading). */
int  ck_group_publishes(ck_handle* h);
int  ck_fetch_groups(ck_handle* h, uint32_t* host_order, uint32_t* host_key_counts, int wait);

/* Kafka RecordBatch v2 framing on the device (reference: aiokafka under broker.subscriber / broker.publish,
 * calfkit/worker/worker.py:45-53, calfkit/nodes/base.py:82-87).  ck_submit_recordbatch takes a fetch response's record set
 * (concatenated v2 frames, uncompressed, gzip, snappy, LZ4 or zstd, below) as it came off the socket: one H2D copy (the frame index goes through page-locked
 * staging the handle owns: nothing waits for the stream), then CRC32C verification, record split and
 * zig-zag varint field decode on the device; the walker reads each value where it lies.  Records of a frame that fails the
 * CRC / framing check get status 6 (bad frame); a truncated trailing frame is ignored.  *n_records = records decoded.
 * ck_fetch_rb_index: per record, where value / key / the `correlation_id` header lie in the submitted buffer (-1 = absent).
 * ck_encode_recordbatch: the publishes host_idx[0..n) of the current plan (one topic-partition, in send order) -> one
 * uncompressed v2 frame (offsetDelta = position in the list, key = correlation id when keyed, headers content-type and
 * correlation_id, CRC32C), built on the device and copied to host_frame. */
int  ck_submit_recordbatch(ck_handle* h, const uint8_t* host_buf, uint64_t nbytes, uint32_t* n_records);
int  ck_fetch_rb_index(ck_handle* h, int64_t* val_off, uint32_t* val_len, int64_t* key_off, int32_t* key_len,
                       int64_t* corr_off, int32_t* corr_len, uint32_t* bad);
/* the same copies queued only (page-locked destinations, ck_sync before reading): the lanes bring the record index back
 * with the step's results (Worker consuming fetch responses, worker/worker.py:45-53) */
int  ck_fetch_rb_index_async(ck_handle* h, int64_t* val_off, uint32_t* val_len, int64_t* key_off, int32_t* key_len,
                             int64_t* corr_off, int32_t* corr_len, uint32_t* bad);
/* LZ4 batches (attributes & 7 = 3) in a fetch response are decoded on the device: each one's records section, one LZ4
 * frame (any block size, linked or independent blocks, block / content checksums and content size verified when present;
 * no dictionary id), lands in a slot behind the raw bytes, and the value / key / correlation_id offsets of its records
 * point there.  A frame that is malformed in any way, or whose block chain runs past the batch, gets status 6 like a CRC
 * failure.  gzip batches (attributes & 7 = 1) are inflated the same way: the records section is one gzip member (RFC 1952
 * / 1951, exactly what zlib's inflate accepts, FHCRC and the trailer's CRC32 and ISIZE checked) inflated into a slot of
 * its ISIZE; a malformed member, or anything after it (a second member included), gets status 6.  zstd batches
 * (attributes & 7 = 4) are decoded the same way: the records section is one zstd frame (RFC 8878, what libzstd 1.5.5
 * accepts with default parameters: window up to 2^27 + 1, no dictionary, content size and XXH64 checksum verified when
 * present) decoded into a slot of the bound the host's walk of its block headers gives (raw and RLE blocks their size,
 * compressed blocks the block maximum, even when the frame states a smaller content size: the literals are decoded into
 * the end of that room); a malformed frame, a skippable or second frame, or anything after the frame gets status 6.
 * Snappy batches (attributes & 7 = 2) are decoded the same way, a warp per chunk: the records section is snappy-java's
 * framing (longer than 16 bytes, magic 82 'SNAPPY' 00, two version words, then big-endian u32 lengths each followed by
 * one raw snappy block, tiling the section) or else one raw snappy block; each block (what Google snappy's RawUncompress
 * accepts) decodes into its place in a slot of exactly the blocks' summed declared lengths.  A section whose chunks do not
 * tile it, a block that snappy refuses or that declares more than 22 times its size, gets status 6.
 * ck_fetch_rb_decoded_async: where those slots start in value-offset space (*base) and their bytes (*nbytes; 0 for a fetch
 * without a gzip, snappy, LZ4 or zstd batch), known as soon as ck_submit_recordbatch returns; with dst given (page-locked, cap >= *nbytes) their
 * D2H copy is queued: value offset v >= *base lies at dst[v - *base] after ck_sync. */
int  ck_fetch_rb_decoded_async(ck_handle* h, uint8_t* dst, uint64_t cap, uint64_t* base, uint64_t* nbytes);
/* Transactions (message format v2, KIP-98; the rule is in csrc/ck_txn.h).  Records a consumer does not deliver get status 7
 * (skipped), val_len 0 and bad = 2 in ck_fetch_rb_index; bad = 1 still means a bad frame.  ck_submit_recordbatch skips
 * every control batch (attributes bit 5) at both isolation levels after checking its CRC32C and its one record's key on
 * the host; a malformed control batch (a bad CRC, a codec, recordsCount != 1, a key shorter than 4 bytes or of negative
 * version) gets status 6, where the Java consumer raises.  Under read_committed the caller computes the mask of the whole
 * fetch once with ck_fetch_txn_mask (no handle, no device): mask[b] = 1 for each complete batch b that is a transactional
 * batch (attributes bit 4) of an aborted producer.  Partition r of the record set is the run of batches starting in
 * [run_start[r], run_start[r + 1]); its aborted transactions (the fetch response's AbortedTransactions list) are the k
 * with abort_run[k] = r, (abort_pid[k], abort_first[k]).  *nbatches = complete batches; fails when cap is smaller, the
 * run starts decrease or an entry names no run.  ck_set_fetch_hidden hands a mask (a slice of it, when the fetch is split
 * at batch boundaries over several handles) to the next ck_submit_recordbatch of the handle, which fails unless nbatches
 * is the number of complete batches it finds; its flagged batches pass the CRC check and are neither decoded nor split.
 * The broker never returns data past a partition's last stable offset to a read_committed fetch: a transaction still
 * open there is the broker's concern, not this one's. */
int  ck_set_fetch_hidden(ck_handle* h, const uint8_t* mask, uint32_t nbatches);
int  ck_fetch_txn_mask(const uint8_t* buf, uint64_t nbytes, const uint64_t* run_start, uint32_t nruns,
                       const uint32_t* abort_run, const int64_t* abort_pid, const int64_t* abort_first, uint32_t naborts,
                       uint8_t* mask, uint32_t cap, uint32_t* nbatches);
/* ck_fetch_positions (no handle, no device): the offsets a consumer of a fetch, or of a slice of one cut at batch
 * boundaries, resumes from.  With the partition runs of ck_fetch_txn_mask, next[r] (nruns entries) = lastOffset + 1
 * (baseOffset + lastOffsetDelta + 1) of the last complete batch starting in run r, -1 when none does; batch_next[b] (cap
 * entries; may be null) the same of each complete batch.  Every batch advances its partition's position, whether it is
 * delivered, skipped (control, aborted) or bad (framing, CRC32C): only the 61-byte headers are read.  *nbatches = complete
 * batches; fails when the run starts decrease or batch_next is shorter. */
int  ck_fetch_positions(const uint8_t* buf, uint64_t nbytes, const uint64_t* run_start, uint32_t nruns,
                        int64_t* next, int64_t* batch_next, uint32_t cap, uint32_t* nbatches);
int  ck_encode_recordbatch(ck_handle* h, const uint32_t* host_idx, uint32_t n, int64_t base_offset, int64_t timestamp_ms,
                           uint8_t* host_frame, uint64_t cap, uint64_t* frame_len);
/* produce side for a whole step (reference: the producer aiokafka runs under broker.publish, nodes/base.py:82-87, and under the
 * handler's publisher, worker/worker.py:52-53, accumulates one record batch per topic-partition).
 *   ck_set_frame_topics       registered topic ids whose publishes are framed (replaces the previous set)
 *   ck_encode_frames          every live publish of the current plan to a frame topic, grouped by (topic, partition) in a
 *                             stable order (records keep their send order; unkeyed publishes form the group of partition -1
 *                             of their topic), split into frames of at most 61 + frame_bytes + one record bytes (ck_set_option
 *                             2, default 1 MiB; rule in DESIGN.md), encoded as ck_encode_recordbatch does with baseOffset 0
 *                             and baseTimestamp timestamp_ms.  Queued only: nothing waits for the host.
 *   ck_encode_frames_records  the same for n records a host path produced for one topic: blob + desc[n][6] = {value off, len,
 *                             key off, len, correlation id off, len} (len -1: absent; key and id as JSON string content,
 *                             unescaped on the device); partition = murmur2(key) % num_partitions as for the plan's publishes
 *   ck_frames_size            frames and bytes of the last pass (waits; frames that did not fit the frame buffer are
 *                             written again into a buffer grown to their size)
 *   ck_fetch_frames_async     frame table and frame bytes of the last pass, queued into page-locked memory (ck_sync);
 *                             ck_frames_size must have been called since the pass */
int  ck_set_frame_topics(ck_handle* h, const int32_t* topic_ids, uint32_t n);
int  ck_encode_frames(ck_handle* h, int64_t timestamp_ms);
int  ck_encode_frames_records(ck_handle* h, int32_t topic_id, const uint8_t* host_blob, uint64_t nbytes, const int64_t* host_desc,
                              uint32_t n, int64_t timestamp_ms);
int  ck_frames_size(ck_handle* h, uint32_t* n_frames, uint64_t* nbytes);
int  ck_fetch_frames_async(ck_handle* h, ck_frame* host_table, uint32_t table_cap, uint8_t* host_frames, uint64_t cap);

/* Idempotent and transactional produce (KIP-98; the Java producer's enable.idempotence and transactional.id).
 *   ck_set_producer           the producer fields of the frames the following passes build (ck_encode_frames,
 *                             ck_encode_frames_records, ck_encode_recordbatch; LZ4 frames too).  flags 0 (the default):
 *                             producerId -1, producerEpoch -1, attributes bit 4 clear.  CK_PRODUCER_IDEMPOTENT: pid and epoch
 *                             (both >= 0); | CK_PRODUCER_TRANSACTIONAL: and attributes bit 4 on every frame.  baseSequence
 *                             stays -1: frames of different passes and handles reach a partition in an order only the host
 *                             knows, so the host writes each frame's baseSequence when it hands the frame out and patches the
 *                             CRC32C with ck_crc32c_patch.  A pass takes the fields when it is queued; the rewrite
 *                             ck_frames_size makes into a grown buffer writes the same headers.
 *   ck_set_sticky_partitions  parts[topic id] (ids < n) the partition the topic's unkeyed publishes join in the following
 *                             passes, -1 none (n = 0: none at all, the default).  The unkeyed publishes are then grouped,
 *                             split and written with that partition's keyed ones, as if they had that partition (Kafka's
 *                             uniform sticky partitioner; an idempotent sequence exists only per partition).  Each entry is
 *                             -1 or in [0, num_partitions).
 *   ck_crc32c_patch           *crc = the CRC32C of a span of len bytes whose CRC32C was *crc, after its 4 bytes at pos changed
 *                             from old4 to new4: O(log len), no handle, no device.  For a frame: span = [21, length), the
 *                             baseSequence at 53 - 21 = 32 of it.
 *   ck_encode_control_batch   the transaction marker the broker appends to a partition when producer (producer_id,
 *                             producer_epoch) commits (type 1) or aborts (type 0): a 78-byte control batch (attributes 0x30,
 *                             baseSequence -1, one record: key version 0 and type, value version 0 and coordinatorEpoch 0),
 *                             CRC32C included, into out (cap >= 78); no handle, no device */
enum { CK_PRODUCER_IDEMPOTENT = 1, CK_PRODUCER_TRANSACTIONAL = 2 };
int  ck_set_producer(ck_handle* h, int64_t pid, int16_t epoch, uint32_t flags);
int  ck_set_sticky_partitions(ck_handle* h, const int32_t* parts, uint32_t n);
int  ck_crc32c_patch(uint32_t* crc, uint64_t len, uint64_t pos, const uint8_t* old4, const uint8_t* new4);
int  ck_encode_control_batch(int64_t base_offset, int64_t timestamp_ms, int64_t producer_id, int16_t producer_epoch, int16_t type,
                             uint8_t* out, uint64_t cap, uint64_t* len);

/* tool node, host tools only: gather every record's tool-call `args` JSON into the output buffer
 * (payload i = args of record i, empty when the record does not reach the tool). */
int  ck_tool_args(ck_handle* h);
/* tool node: run + publish plan + encode + route.  host_aux/host_aux_off: JSON return values per
 * record (offsets[n+1]) for host tools, NULL for a device template. */
int  ck_tool_plan(ck_handle* h, const uint8_t* host_aux, const int64_t* host_aux_off);
/* ReturnCall of the state as it is on the wire (e.g. an Agent's final output after the host LLM step):
 * pop the current frame, publish to its callback topic and to the node's publish_topic. */
int  ck_return_plan(ck_handle* h);
/* client reply path (calfkit/client/deserialize.py:55-89): payload i = the output value of reply envelope i as JSON —
 * mode 0: first DataPart.data of final_output_parts, else first TextPart.text (auto); 1: TextPart.text only
 * (output_type=str); 2: DataPart.data only (typed output; the caller validates the value).  A reply without the
 * wanted part (the reference raises DeserializationError) gets CK_ACT_RAISES and an empty payload.  No publishes. */
int  ck_reply_plan(ck_handle* h, uint32_t mode);
/* same as ck_tool_plan, aux blob already in HBM */
int  ck_tool_plan_device(ck_handle* h, const uint8_t* dev_aux, const int64_t* dev_aux_off);

/* agent fan-out (calfkit/nodes/agent.py:177-211 + nodes/base.py:73-88): one Call envelope per
 * pending tool call of every record.  tool_names/topic strings: registry tool_name -> subscribe
 * topic[0]; agent_name/callback: the agent's name and subscribe_topics[0]; frame ids are uuid7s
 * built from (unix_ms, seed, output index). */
int  ck_set_agent_node(ck_handle* h, int32_t publish_topic_id, const uint8_t* agent_name, uint32_t agent_name_len,
                       const uint8_t* callback_topic, uint32_t callback_len,
                       const uint8_t* tool_names, const uint32_t* tool_name_off,
                       const uint8_t* tool_topics, const uint32_t* tool_topic_off, uint32_t ntools);
int  ck_set_agent_tool_topic_ids(ck_handle* h, int32_t self_topic_id /* id of the agent's subscribe_topics[0], -1 = unregistered */,
                                 const uint32_t* ids /* 0xffffffff = unregistered */, uint32_t ntools);
/* sequential != 0: Agent(sequential_only_mode=True) — only the first pending call goes out, as a single
 * Call (agent.py:94-108,179-192). */
int  ck_fanout_plan(ck_handle* h, uint64_t unix_ms, uint64_t seed, uint32_t max_fanout, uint32_t sequential);
/* TailCall to the agent's own topic (all requested tools invalid -> retry, agent.py:171-175;
 * nodes/base.py:120-136): the current frame is replaced by a fresh one inheriting its callback_topic. */
int  ck_tailcall_plan(ck_handle* h, uint64_t unix_ms, uint64_t seed);
/* aggregation gate on the device (calfkit/nodes/agent.py:57-68 _parallel_state_aggregation, models/state.py:127-141
 * PendingToolBatch): an HBM-resident table keyed by correlation id holding, per pending fan-out, the state the agent fanned
 * out from and the expected tool_call_ids with the results collected so far.
 *   ck_gate_create    sizes the table (entries = concurrent fan-outs, slots = sum of their expected ids, arena < 4 GiB);
 *                     entries, slots and arena are allocated twice (the second set is what ck_gate_compact moves into)
 *   ck_gate_register  after ck_fanout_plan on a batch of post-LLM envelopes: every record that went out as list[Call]
 *                     (ACTION == CK_ACT_FANOUT) becomes a pending entry (a new one replaces an old one for the same id;
 *                     within one batch the highest record index wins).  A fan-out that finds no room is not registered
 *                     and counted as a failure: its tool returns pass through
 *   ck_gate_arrive    on a submitted batch of records arriving at the agent's topic; stamp_base = records this node
 *                     consumed before this batch (arrival order across and inside batches).  Column ACTION afterwards:
 *                     CK_ACT_SILENT (collected, still incomplete; only the handler-return publish to publish_topic),
 *                     9 = complete (payload i = inbound envelope carrying base_state + the collected results in order
 *                     of collection; the entry is deleted), 10 = no pending fan-out (continue with the inbound state).
 *                     A completing record whose results found no room in the arena is declined (STATUS CK_UNSUPPORTED,
 *                     ACTION CK_ACT_RAISES), counted as a failure, and its entry is deleted
 *   ck_gate_stats     out5 = {entries used, slots used, arena bytes used, live entries, capacity failures of the last
 *                     register / arrive call}
 *   ck_gate_compact   moves the live entries to fresh space and rebuilds the key table: gives back what finished
 *                     fan-outs used (run it when entries, slots or arena bytes used pass a threshold)
 *   ck_gate_reset     forget everything */
int  ck_gate_create(ck_handle* h, uint32_t max_entries, uint32_t max_slots, uint64_t arena_bytes);
int  ck_gate_register(ck_handle* h, uint32_t min_pending /* 2 = the reference's rule; 1 also registers single Calls */);
int  ck_gate_arrive(ck_handle* h, uint64_t stamp_base);
int  ck_gate_stats(ck_handle* h, uint64_t* out5);
int  ck_gate_compact(ck_handle* h);
int  ck_gate_reset(ck_handle* h);
/* cross-partition forward over NVLink peer memory (records shard by Kafka partition across the GPUs of a box; reference
 * analogue: producing to a topic-partition another worker process consumes, nodes/base.py:82-87 key=correlation_id).
 *   ck_comm_create    this rank's receive buffer: one region per source rank (max_fwd payloads, data_cap bytes each);
 *                     ipc_handle_out[64] is handed to every peer (any side channel); max_fwd and data_cap MUST be the same
 *                     on every rank (a rank addresses its region inside a peer's buffer with its own geometry)
 *   ck_comm_connect   handles[world][64] in rank order: maps the peers' receive buffers (CUDA IPC, same box)
 *   ck_exchange_send  plan + pack + transfer in one pass on the handle's stream, no host synchronisation: the keyed
 *                     publishes of the current plan whose partition % world != rank are written straight into the owner's
 *                     region for this rank (payload bytes 16-byte aligned + {len, topic_id, partition, source publish}),
 *                     then the region header {step, count, overflow, bytes}.  The caller brackets it with two barriers:
 *                     before (every peer has consumed what it received last time) and after (all stores have landed).
 *   ck_recv_info / ck_fetch_received: where the regions are / one region copied to the host */
int  ck_comm_create(ck_handle* h, uint32_t rank, uint32_t world, uint32_t max_fwd, uint64_t data_cap, uint8_t* ipc_handle_out);
int  ck_comm_connect(ck_handle* h, const uint8_t* handles);
int  ck_exchange_send(ck_handle* h, uint64_t step);
int  ck_recv_info(ck_handle* h, void** dev_recv, uint64_t* region_stride, uint32_t* max_fwd, uint64_t* data_cap);
int  ck_fetch_received(ck_handle* h, uint32_t src, uint64_t* hdr4, uint8_t* host_meta, uint8_t* host_data, uint64_t data_cap);
/* pipelined form: ck_peek_received reads all region headers ([world][4] = step, count, overflow, nbytes) with one stream
 * synchronisation; ck_fetch_received_async queues the copies of region `src` into page-locked memory and returns (complete
 * after the next ck_sync).  A region stays valid until this engine's next ck_exchange_send. */
int  ck_peek_received(ck_handle* h, uint64_t* hdr4);
int  ck_fetch_received_async(ck_handle* h, uint32_t src, uint64_t count, uint64_t nbytes, uint8_t* host_meta, uint8_t* host_data);
/* multi-GPU exchange planning (records shard by Kafka partition across the GPUs of a box; reference analogue:
 * producing to a topic-partition another worker process consumes, nodes/base.py:82-87 key=correlation_id).  Selects the
 * keyed publishes whose partition % world != rank, ordered by destination rank (stable), into library-owned device
 * arrays: payload span in the output buffer (src_off, len), offset in the packed send buffer (dst_off, exclusive
 * scan of len) and the index of the publish (pub).  host_counts / host_nbytes [world]: payloads and bytes per
 * destination (the all-to-all split sizes).  Waits for the stream once. */
int  ck_exchange_plan(ck_handle* h, uint32_t rank, uint32_t world, const int64_t** dev_src_off, const int64_t** dev_len,
                      const int64_t** dev_dst_off, const uint32_t** dev_pub, int64_t* host_counts, int64_t* host_nbytes,
                      uint32_t* n_sel);

/* results ---------------------------------------------------------------------------------------- */
int  ck_sync(ck_handle* h);
uint64_t ck_launch_count(ck_handle* h);   /* kernels launched by this handle so far */
int  ck_out_size(ck_handle* h, uint64_t* out_bytes, uint32_t* n_payloads, uint32_t* n_publishes);  /* waits */
int  ck_fetch_columns(ck_handle* h, uint32_t* host_cols /* CK_NUM_COLS * n, column-major */);
/* records of the current batch that were not in the canonical spelling (re-emitted into the overlay, or rejected), and the
 * overlay bytes in use; 0 / 0 means every column span refers to the submitted bytes */
int  ck_canon_stats(ck_handle* h, uint32_t* n_listed, uint64_t* overlay_bytes);
/* k selected rows of the column table: host_rows[j * n + i] = column which[j] of record i */
int  ck_fetch_cols(ck_handle* h, const uint32_t* which, uint32_t k, uint32_t* host_rows);
/* page-locked host memory for batch arenas: the landing zone of polled record batches (reference seam: the consume loop
 * FastStream runs under calfkit/worker/worker.py:45-51) and of the produced payloads; copies to and from it overlap with
 * the kernels and with each other.  ck_last_error(NULL) after a failure. */
int  ck_host_alloc(uint64_t bytes, void** out);
void ck_host_free(void* p);
/* payload i = host_out[host_out_off[i] .. + host_out_len[i]); starts are 16-byte aligned, so
 * host_out_off[i+1] - host_out_off[i] is the length rounded up to 16 and *out_bytes of ck_out_size is
 * the padded total */
int  ck_fetch_output(ck_handle* h, uint8_t* host_out, uint64_t cap, int64_t* host_out_off /* n_payloads+1 */,
                     uint32_t* host_out_len /* n_payloads */, ck_publish* host_pubs /* n_publishes */);
/* the same copies queued only (page-locked destinations): overlap host work, then ck_sync before reading */
int  ck_fetch_output_async(ck_handle* h, uint8_t* host_out, uint64_t cap, int64_t* host_out_off, uint32_t* host_out_len,
                           ck_publish* host_pubs);
int  ck_fetch_cols_async(ck_handle* h, const uint32_t* which, uint32_t k, uint32_t* host_rows);
/* canonical re-emissions of the records that were submitted in a non-canonical spelling: record i has one iff
 * host_off[i] >= 0 (then host_ovl[host_off[i] .. + host_len[i]) are its canonical bytes; column spans of that
 * record refer to them) */
int  ck_fetch_overlay(ck_handle* h, uint8_t* host_ovl, uint64_t cap, int64_t* host_off, uint32_t* host_len, uint64_t* used);
int  ck_fetch_topic_hist(ck_handle* h, uint32_t* host_hist, uint32_t n);

/* introspection for benchmarks / tests ------------------------------------------------------------ */
void* ck_stream(ck_handle* h);                     /* cudaStream_t of the handle */
int  ck_device_buffers(ck_handle* h, void** in, void** in_off, void** out, void** out_off, void** cols);
int  ck_device_buffers2(ck_handle* h, void** pubs, void** pay_len, void** descs);
int  ck_profile(ck_handle* h, int enable);         /* record (asynchronous) CUDA events around every kernel */
int  ck_profile_read(ck_handle* h, float* ms /* CK_NUM_KERNELS */, uint32_t* launches /* CK_NUM_KERNELS */, int reset);

enum { CK_K_WALK = 0, CK_K_PLAN, CK_K_SCAN, CK_K_EMIT, CK_K_ROUTE, CK_K_FANOUT, CK_K_CANON, CK_K_WALK_LONG, CK_K_WALK_ELEMS, CK_K_FRAME, CK_K_LZ4, CK_NUM_KERNELS };

#ifdef __cplusplus
}
#endif
#endif
