// Shared definitions for the calfkit-b200 device code and its C-ABI (plain C compatible).
#ifndef CK_COMMON_H
#define CK_COMMON_H

#include <stdint.h>

// ---------------------------------------------------------------------------------------------
// Per-record decode status (column CK_COL_STATUS).  Mirrors the error classes pydantic reports for
// Envelope.model_validate_json (reference calfkit/models/envelope.py:9-17; SURVEY.md Appendix A):
// a bad record never fails the batch.
// ---------------------------------------------------------------------------------------------
enum {
    CK_OK = 0,               // valid Envelope AND byte-wise a fixed point of dump(validate(.)) -> splice path
    CK_NOT_CANONICAL = 1,    // well-formed so far but not a recognised fixed point (needs the canonicaliser)
    CK_JSON_INVALID = 2,     // pydantic: json_invalid
    CK_SCHEMA_INVALID = 3,   // pydantic: missing / string_type / union_tag_invalid / ... (detail in CK_COL_ERR)
    CK_UNSUPPORTED = 4,      // valid-looking but uses a construct the device path does not handle yet
    CK_EMPTY = 5,            // zero-length record
    CK_BAD_FRAME = 6         // the Kafka record batch that carried it failed the CRC32C / framing check (ck_submit_recordbatch)
};

// What the node does with the record (column CK_COL_ACTION), reference nodes/base.py:70-147.
enum {
    CK_ACT_NONE = 0,         // rejected record: nothing is published
    CK_ACT_RETURN = 1,       // ReturnCall: pop frame, publish to callback_topic (+ handler return to publish_topic)
    CK_ACT_SILENT = 2,       // Silent: only the handler-return publish (input bytes) to publish_topic
    CK_ACT_RAISES = 3,       // the reference handler raises (e.g. input_args null for a tool node): no publish
    CK_ACT_CALL = 4,         // Call: push frame, publish to target
    CK_ACT_TAILCALL = 5,     // TailCall: pop + push inheriting callback
    CK_ACT_FANOUT = 6,       // list[Call]: one publish per pending tool call; handler return = input
    CK_ACT_HOST_TOOL = 7,    // tool result must come from the host (tool is not a device template)
    CK_ACT_REPLY = 8,        // client reply: the payload is the output value (DataPart.data / TextPart.text as JSON)
    CK_ACT_GATE_COMPLETE = 9,// aggregation gate: this arrival completed its fan-out; payload = envelope carrying the merged state
    CK_ACT_GATE_PASS = 10    // aggregation gate: no pending fan-out for this correlation id
};

// ---------------------------------------------------------------------------------------------
// Columnar event table: one uint32 column per field, `max_records` entries each (SoA, so a warp of
// 32 records writes 128 contiguous bytes per column).  Offsets are relative to the record start.
// ---------------------------------------------------------------------------------------------
enum {
    CK_COL_STATUS = 0,
    CK_COL_ACTION,
    CK_COL_ERR,              // position (byte offset) where recognition stopped, for diagnostics
    CK_COL_CORR_OFF, CK_COL_CORR_LEN,             // deps.correlation_id (string content, raw JSON bytes)
    CK_COL_NFRAMES,
    CK_COL_FRAMES_OFF, CK_COL_FRAMES_LEN,         // call_stack._internal_list value span, brackets included
    CK_COL_TOP_OFF, CK_COL_TOP_LEN,               // last frame object span
    CK_COL_TGT_OFF, CK_COL_TGT_LEN,               // top frame target_topic content
    CK_COL_CB_OFF, CK_COL_CB_LEN,                 // top frame callback_topic content
    CK_COL_NARGS,                                 // top frame input_args: 0xffffffff = null, else element count
    CK_COL_ARG0_OFF, CK_COL_ARG0_LEN,             // element 0 span (content if string, whole value otherwise)
    CK_COL_ARG1_OFF, CK_COL_ARG1_LEN,
    CK_COL_ARGKINDS,                              // bit0: arg0 is a string, bit1: arg1 is a string
    CK_COL_FOV_OFF, CK_COL_FOV_LEN,               // top frame overrides value span ("null" or object)
    CK_COL_TC_OFF, CK_COL_TC_LEN,                 // state.tool_calls value span
    CK_COL_TR_OFF, CK_COL_TR_LEN,                 // state.tool_results value span
    CK_COL_UNC_OFF, CK_COL_UNC_LEN,               // state.uncommitted_message
    CK_COL_HIST_OFF, CK_COL_HIST_LEN,             // state.message_history
    CK_COL_FOP_OFF, CK_COL_FOP_LEN,               // state.final_output_parts
    CK_COL_TI_OFF, CK_COL_TI_LEN,                 // state.temp_instructions
    CK_COL_SMETA_OFF, CK_COL_SMETA_LEN,           // state.metadata
    CK_COL_SOV_OFF, CK_COL_SOV_LEN,               // state.overrides
    CK_COL_PD_OFF, CK_COL_PD_LEN,                 // deps.provided_deps
    CK_COL_WFMETA_OFF, CK_COL_WFMETA_LEN,         // internal_workflow_state.metadata
    // filled by the tool-node plan kernel
    CK_COL_CALL_VAL_OFF, CK_COL_CALL_VAL_LEN,     // tool_calls[arg0] value span (the ToolCallPart object)
    CK_COL_TNAME_OFF, CK_COL_TNAME_LEN,           // its tool_name content
    CK_COL_ARGS_OFF, CK_COL_ARGS_LEN,             // its args value span
    CK_COL_RES_OFF, CK_COL_RES_LEN,               // existing tool_results[arg0] value span (len 0 = absent)
    CK_COL_NOUT,                                  // number of publishes this record produces
    // client reply path (reference client/deserialize.py:55-89): the output of a final reply
    CK_COL_ODATA_OFF, CK_COL_ODATA_LEN,           // first DataPart of final_output_parts: its `data` value span (len 0 = none)
    CK_COL_OTEXT_OFF, CK_COL_OTEXT_LEN,           // first TextPart: its `text` JSON string span, quotes included (len 0 = none)
    CK_NUM_COLS
};

#define CK_NARGS_NULL 0xffffffffu

// Output-record descriptor written by the plan kernels and consumed by emit/route.
// An output payload is the concatenation of up to CK_MAX_SEGS segments.  A segment may start and end at
// any byte of the payload, and may be empty; the payload itself starts 16-byte aligned in the output buffer.
// Every source is readable up to 19 bytes past a segment's end (the emitter reads aligned words).
#define CK_MAX_SEGS 16
enum { CK_SRC_INPUT = 0, CK_SRC_LIT = 1, CK_SRC_AUX = 2, CK_SRC_GLUE = 3 };   // input record / literal pool / per-batch aux blob / per-payload glue slot
#define CK_GLUE_STRIDE 512    // bytes of scratch per payload in which a plan thread assembles the new text of a splice
typedef struct {
    uint32_t nseg;
    uint32_t record;                 // index of the input record this output derives from
    uint32_t total_len;
    uint32_t pad;
    uint32_t seg[CK_MAX_SEGS][2];    // {offset inside the source (INPUT: relative to the record start), (len << 2) | src}
} ck_out_desc;                       // 144 B; a payload with n segments occupies the first 16 + 8 n bytes

#endif
