/*
 * mashmap_b200_align.h -- C ABI of the device path of mashmap-b200-align (base-level alignment of mappings).
 *
 * The reference aligner (src/align, mashmap-align) calls edlibAlign(query, target, k, EDLIB_MODE_HW, EDLIB_TASK_PATH)
 * once per mapping line on one CPU thread (computeAlignments.hpp:268-269). These entry points run that call for a whole
 * batch of mappings on the device and give the same edit distance, start, end and edit-op path (DESIGN.md section 10).
 * They also run edlib's global mode (EDLIB_MODE_NW), which mashmap-b200 --align uses for the exact PAF region.
 * Same conventions as mashmap_b200.h: MM_OK or a negative MM_E* code, mm_align_last_error() for the text, no CPU
 * fallback. Lives in libmashmap_b200.so.
 */
#ifndef MASHMAP_B200_ALIGN_H
#define MASHMAP_B200_ALIGN_H

#include <stdint.h>

#include "mashmap_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Alignment modes of a job (edlib's EdlibAlignMode). */
#define MM_ALIGN_HW 0 /* EDLIB_MODE_HW: the query anywhere in the target (mashmap-b200-align)                         */
#define MM_ALIGN_NW 1 /* EDLIB_MODE_NW: query and target end to end (mashmap-b200 --align); start 0, end t_len - 1 */

/* Routing of NW sub-problems: the NW distance of an MM_ALIGN_NW job and every Hirschberg node (both modes) whose
 * max(query length, target length) is at least this run banded, one CTA per sweep; shorter ones run unbanded, one warp
 * per problem. Both give edlib's results (DESIGN.md section 10); the rule reads only the sub-problem's own size. */
#define MM_ALIGN_BAND_MIN_LEN (32 * 1024)

/* One edlibAlign call: query = qbases[q_offset, q_offset + q_len) (already oriented: the reverse complement for a '-'
 * mapping, computeAlignments.hpp:243-248), target = tbases[t_offset, t_offset + t_len) (:230-236), and
 * k = editDistanceLimit (:256-261; k < 0: unbounded, edlib's doubling from 64, edlib.hxx:173-191). Bytes are compared for
 * identity only (no additional equalities): N matches N, NUL matches NUL. q_len, t_len >= 1. mode: MM_ALIGN_HW or
 * MM_ALIGN_NW (anything else is MM_EINVAL); a batch may mix them, and a job's result does not depend on the others.
 * 32 bytes. */
typedef struct mm_align_job {
  uint64_t q_offset;
  uint64_t t_offset;
  int32_t q_len;
  int32_t t_len;
  int32_t k;
  int32_t mode;
} mm_align_job;

/* EdlibAlignResult for one job (edlib.h:178-228): ed = editDistance (-1: none within k), start / end =
 * startLocations[0] / endLocations[0] (target coordinates, end inclusive; end = -1 with start = 0 for the path that
 * inserts the whole query), alignment_length and the path as edit ops (EDLIB_EDOP_*: 0 match, 1 insertion, 2 deletion,
 * 3 mismatch) at ops[ops_offset, ops_offset + alignment_length). 24 bytes. */
typedef struct mm_align_result {
  int32_t ed;
  int32_t start;
  int32_t end;
  int32_t alignment_length;
  uint64_t ops_offset;
} mm_align_result;

typedef struct mm_align_ctx mm_align_ctx;

/* Replaces nothing in the reference (it has no device). scratch_bytes bounds the device memory one batch's kernels
 * use beyond the inputs and the op buffer (0: half the free memory, at most 8 GiB); work that does not fit runs in
 * waves. */
int mm_align_ctx_create(int device, uint64_t scratch_bytes, mm_align_ctx **out);
int mm_align_ctx_destroy(mm_align_ctx *ctx);
const char *mm_align_last_error(const mm_align_ctx *ctx); /* ctx may be NULL: error of the last failed create */

/* edlibAlign(job.mode, PATH) (edlib.hxx:141-260) for every job: qbases / tbases in host memory (pinned or not, see
 * mm_host_alloc). results[n_jobs]; ops[ops_cap]. On MM_ECAPACITY *n_ops holds the op count needed and nothing else is
 * valid; the sum of q_len + t_len over the jobs is always enough. A batch may hold at most 16 distinct byte values. */
int mm_align_batch(mm_align_ctx *ctx, const char *qbases, uint64_t n_qbases, const char *tbases, uint64_t n_tbases,
                   const mm_align_job *jobs, uint64_t n_jobs, mm_align_result *results, uint8_t *ops,
                   uint64_t ops_cap, uint64_t *n_ops);

/* CUDA-event time in milliseconds of each stage of the last mm_align_batch or mm_align_batch_tags:
 * [0] H2D  [1] distance and end (HW and NW passes)  [2] start (reverse SHW pass)  [3] Hirschberg levels  [4] leaf NW + traceback
 * [5] D2H  [6] whole call on the host clock  [7] number of Hirschberg levels. */
int mm_align_last_stage_ms(const mm_align_ctx *ctx, float ms[8]);

/* Flags of mm_align_batch_tags. 0: cg is edlibAlignmentToCigar(EDLIB_CIGAR_STANDARD), runs of M, I, D.
 * MM_ALIGN_TAG_EQX: cg is edlibAlignmentToCigar(EDLIB_CIGAR_EXTENDED), runs of = (op 0), X (3), I (1), D (2).
 * MM_ALIGN_TAG_CS: also minimap2's short cs: ":N" per match run, "*tq" per mismatch (target byte, then query byte),
 * "+bases" / "-bases" per insertion / deletion run; bases are the job's bytes with A-Z lowered to a-z. */
#define MM_ALIGN_TAG_EQX (1u << 0)
#define MM_ALIGN_TAG_CS (1u << 1)

/* One job of mm_align_batch_tags: ed and alignment_length as in mm_align_result; the cg body (no "cg:Z:") at
 * text[cg_offset, cg_offset + cg_len) and, with MM_ALIGN_TAG_CS, the cs body at text[cs_offset, cs_offset + cs_len).
 * Lengths are 0 for a job with no path (ed < 0 or alignment_length 0). 40 bytes. */
typedef struct mm_align_tag_result {
  int32_t ed;
  int32_t alignment_length;
  uint64_t cg_offset;
  uint64_t cg_len;
  uint64_t cs_offset;
  uint64_t cs_len;
} mm_align_tag_result;

/* The alignment of mm_align_batch (same distance, same path) for MM_ALIGN_NW jobs only (any other mode is MM_EINVAL),
 * returned as tag text written on the device instead of edit ops. flags: 0 or MM_ALIGN_TAG_EQX, optionally with
 * MM_ALIGN_TAG_CS (other bits are MM_EINVAL). text[text_cap]; on MM_ECAPACITY *n_text holds the text size needed and
 * nothing else is valid. */
int mm_align_batch_tags(mm_align_ctx *ctx, const char *qbases, uint64_t n_qbases, const char *tbases, uint64_t n_tbases,
                        const mm_align_job *jobs, uint64_t n_jobs, uint32_t flags, mm_align_tag_result *results,
                        char *text, uint64_t text_cap, uint64_t *n_text);

/* CUDA-event time in milliseconds of the formatting kernels of the last mm_align_batch_tags (path compaction, runs,
 * text); its text D2H counts in stage [5] of mm_align_last_stage_ms. */
int mm_align_last_tag_ms(const mm_align_ctx *ctx, float *ms);

#ifdef __cplusplus
}
#endif
#endif /* MASHMAP_B200_ALIGN_H */
