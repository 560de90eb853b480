/*
 * mashmap_b200_nccl.h -- multi-GPU entry points of the H100 mapping hot path (libmashmap_nccl.so; links NCCL).
 *
 * The reference (marbl/MashMap v3.1.3) is a single-process CPU program: there is no collective, no device and no
 * rank anywhere in it (SURVEY section 0, fact 5). What it has instead is ONE in-memory index (skch::Sketch, reference
 * src/map/include/winSketch.hpp:57-511) read by every worker thread (ThreadPool.hpp) and ONE ordered stream of
 * mapping results (computeMap.hpp:724-747; with -f one-to-one all results are filtered together, :358-405).
 * These calls are what replaces "every worker sees the same Sketch" and "all results come together" when the
 * workers are GPUs (SURVEY 8(e)):
 *   mm_index_broadcast    the device image of the index goes from the rank that built it to every other rank with
 *                         ONE ncclBroadcast over NVLink / NVSwitch (replaces: const Sketch& shared by the threads);
 *   mm_records_allgather  fixed-size mapping records of all ranks on every rank (one all-gather of counts + one of
 *                         padded records; replaces: the single output queue of ThreadPool / allReadMappings);
 *   mm_index_replicate    the same broadcast inside ONE process that drives several devices (skch::Map --devices).
 * Reads are sharded by contiguous blocks across ranks; there is no collective on the mapping path itself.
 *
 * A communicator is created from a 128-byte NCCL unique id that rank 0 makes (mm_comm_unique_id) and hands to the
 * other ranks by whatever channel the host program has (MPI, a file, torch.distributed ...).
 */
#ifndef MASHMAP_B200_NCCL_H
#define MASHMAP_B200_NCCL_H

#include <stdint.h>

#include "mashmap_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define MM_COMM_ID_BYTES 128

typedef struct mm_comm mm_comm;

/* rank 0: a fresh NCCL unique id (ncclGetUniqueId) */
int mm_comm_unique_id(uint8_t id[MM_COMM_ID_BYTES]);
/* every rank: joins the communicator on `device` (ncclCommInitRank). Collective. */
int mm_comm_create(const uint8_t id[MM_COMM_ID_BYTES], int n_ranks, int rank, int device, mm_comm **out);
int mm_comm_destroy(mm_comm *comm);
const char *mm_comm_last_error(const mm_comm *comm); /* comm may be NULL: error of the last failed create */

/* Collective. `root` owns an index image (mm_index_upload, or an earlier broadcast); every other rank's context
 * receives it and is ready to map afterwards (tables included). Returns the image size in *n_bytes (may be NULL). */
int mm_index_broadcast(mm_ctx *ctx, mm_comm *comm, int root, uint64_t *n_bytes);

/* Collective. records: n_records host records of record_bytes bytes each on this rank. out: host buffer for all
 * ranks' records, rank by rank, in rank order (capacity out_cap_records records); counts[n_ranks] = records per rank.
 * MM_ECAPACITY (with counts filled) if out is too small. */
int mm_records_allgather(mm_comm *comm, const void *records, uint64_t n_records, uint32_t record_bytes,
                         void *out, uint64_t out_cap_records, uint64_t *counts);

/* One process, several devices: the image of `src` is copied to the n_dst contexts (each on its own device) with one
 * grouped ncclBroadcast. */
int mm_index_replicate(mm_ctx *src, mm_ctx *const *dst, int n_dst);

#ifdef __cplusplus
}
#endif
#endif /* MASHMAP_B200_NCCL_H */
